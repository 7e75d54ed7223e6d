"""CPU-only tests of the host side: C-ABI surface, program translation, scheme
assembly, geometry, time-step logic.  No compute call needs a GPU here."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import pysph_b200 as pb
from pysph_b200 import _lib, geometry as geo
from pysph_b200.program import build_program

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, 'include', 'b200sph.h')).read()
    declared = set(re.findall(r'\b(b200sph_[a-z0-9_]+)\s*\(', hdr))
    declared -= {'b200sph_ctx'}
    assert len(declared) >= 25
    lib = _lib.load()
    for name in sorted(declared):
        assert hasattr(lib, name), 'libb200sph.so does not export %s' % name
    # and the ctypes table covers exactly the header
    assert set(_lib.SIGNATURES) == declared
    assert lib.b200sph_abi_version() == 6


def test_no_cpu_fallback_without_device():
    """Without a GPU the product path must fail loudly, not fall back."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        pytest.skip('GPU present')
    pa = pb.get_particle_array_wcsph(name='f', x=np.zeros(4))
    with pytest.raises(_lib.B200Error):
        pb.B200Backend([pa])


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, 'pysph_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.h')):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle', src, re.M), f
                assert 'liboracle' not in src, f


def test_struct_layouts_match_header():
    # sizes implied by include/b200sph.h (x86-64 SysV)
    assert C.sizeof(_lib.PairProgram) == 8 * 8 * 4 + 2 * 4 + 9 * 8
    assert C.sizeof(_lib.TvfProgram) == 4 * 4 + 11 * 8 + 2 * 4 + 8
    assert C.sizeof(_lib.GridInfo) == 8 + 8 + 24 + 24 + 12 + 4 + 8 + 8
    assert C.sizeof(_lib.Stats) == 3 * 8 + 17 * 8
    ids = _lib.PROP_IDS
    assert ids['x'] == 0 and ids['rho'] == 6 and ids['h'] == 7 and ids['m'] == 8
    assert ids['rho0'] == 15 and ids['p'] == 16 and ids['dt_force'] == 26


def test_wcsph_scheme_equations_order():
    # scheme.py:388-506 for dam_break_3d (hg_correction, no update_h)
    s = pb.WCSPHScheme(['fluid'], ['boundary', 'obstacle'], dim=3, rho0=1000.0,
                       c0=32.85, h0=0.026, hdx=1.3, gz=-9.81, alpha=0.25,
                       beta=0.0, gamma=7.0, hg_correction=True)
    groups = s.get_equations()
    assert [g.real for g in groups] == [False, True]
    g1 = [(e.name, e.dest) for e in groups[0].equations]
    assert g1 == [('TaitEOS', 'fluid'), ('TaitEOSHGCorrection', 'boundary'),
                  ('TaitEOSHGCorrection', 'obstacle')]
    g2 = [(e.name, e.dest, e.sources) for e in groups[1].equations]
    assert g2 == [
        ('ContinuityEquation', 'boundary', ['fluid']),
        ('ContinuityEquation', 'obstacle', ['fluid']),
        ('ContinuityEquation', 'fluid', ['fluid', 'boundary', 'obstacle']),
        ('MomentumEquation', 'fluid', ['fluid', 'boundary', 'obstacle']),
        ('XSPHCorrection', 'fluid', ['fluid'])]
    # nu != 0: LaminarViscosity inserted before XSPH (scheme.py:486-496); delta_sph has no kernels
    s = pb.WCSPHScheme(['fluid'], ['boundary'], dim=3, rho0=1000.0, c0=32.85, h0=0.026, hdx=1.3,
                       nu=1e-3)
    g2 = [(e.name, e.sources) for e in s.get_equations()[1].equations]
    assert g2[-2:] == [('LaminarViscosity', ['fluid', 'boundary']), ('XSPHCorrection', ['fluid'])]
    ops = build_program(s.get_equations(), ['fluid', 'boundary'], 3)
    prog = [o for o in ops if o[0] == 'pair'][0][1]
    assert prog.eqmask[0][1] & _lib.EQ_LAMINAR and prog.nu == 1e-3 and prog.eta == 0.01
    with pytest.raises(NotImplementedError):
        pb.WCSPHScheme(['fluid'], [], dim=3, rho0=1000.0, c0=32.85, h0=0.026, hdx=1.3, delta_sph=True)
    with pytest.raises(NotImplementedError):
        pb.WCSPHScheme(['f'], [], dim=2, rho0=1, c0=1, h0=1, hdx=1, delta_sph=True)


def test_program_translation():
    names = ['fluid', 'boundary', 'obstacle']
    s = pb.WCSPHScheme(['fluid'], ['boundary', 'obstacle'], dim=2, rho0=1000.0,
                       c0=62.0, h0=0.039, hdx=1.3, gy=-9.81, alpha=0.1,
                       hg_correction=True, update_h=True)
    ops = build_program(s.get_equations(), names, 2)
    kinds = [o[0] for o in ops]
    assert kinds == ['eos', 'eos', 'eos', 'pair', 'ferrari']
    assert ops[0][1:3] == (0, 0) and ops[1][1:3] == (1, 1) and ops[0][-1] == 0
    prog = ops[3][1]
    F, B, O = 0, 1, 2
    CONT, MOM, XSPH = _lib.EQ_CONTINUITY, _lib.EQ_MOMENTUM, _lib.EQ_XSPH
    assert prog.eqmask[F][F] == CONT | MOM | XSPH
    assert prog.eqmask[F][B] == CONT | MOM and prog.eqmask[F][O] == CONT | MOM
    assert prog.eqmask[B][F] == CONT and prog.eqmask[B][B] == 0
    assert prog.eqmask[O][F] == CONT and prog.eqmask[O][B] == 0
    assert prog.real_only == 1 and prog.gy == -9.81 and prog.alpha == 0.1
    assert prog.eps_xsph == 0.5 and prog.c0 == 62.0
    assert ops[4] == ('ferrari', 0, 1.3, 2, 0)

    # unsupported constructs fail at setup time
    with pytest.raises(NotImplementedError):
        build_program([pb.Group([pb.SummationDensity('fluid', ['fluid']),
                                 pb.XSPHCorrection('fluid', ['fluid'])])],
                      names, 3)
    # the loop nest's control features become nested ops (mako:262-363)
    cond = lambda t, dt: True
    ops = build_program([pb.Group([pb.SummationDensity('fluid', ['fluid'])],
                                  iterate=True, min_iterations=2, max_iterations=5,
                                  condition=cond, start_idx=1, stop_idx='n')],
                        names, 3, particle_arrays=[
                            pb.get_particle_array_wcsph(name=n) for n in names])
    assert ops[0][0] == 'cond' and ops[0][1] is cond
    it = ops[0][2][0]
    assert it[0] == 'iterate' and it[1:3] == (2, 5)
    assert [o[0] for o in it[4]] == ['range', 'pair']
    assert it[4][0][1][0][:2] == (1, 'n') and it[4][1][1].real_only == 0
    with pytest.raises(NotImplementedError):     # ranges: the WCSPH pair equations only
        build_program([pb.Group([pb.TaitEOS('fluid', None, rho0=1., c0=1., gamma=7.)],
                                stop_idx=3)], names, 3)
    with pytest.raises(NotImplementedError):
        build_program([pb.Group([
            pb.MomentumEquation('fluid', ['fluid'], c0=1.0, alpha=0.1),
            pb.MomentumEquation('boundary', ['fluid'], c0=1.0, alpha=0.2)])],
            names, 3)
    with pytest.raises(ValueError):
        build_program([pb.SummationDensity('nope', ['fluid'])], names, 3)
    # a bare list of equations is one Group (equation.py:346-373)
    ops = build_program([pb.SummationDensity('fluid', ['fluid', 'boundary'])],
                        names, 3)
    assert ops[0][0] == 'pair' and ops[0][1].eqmask[0][1] == 1
    # subgroups are flattened in order, update_nnps is honoured
    ops = build_program([pb.Group([
        pb.Group([pb.SummationDensity('fluid', ['fluid'])], update_nnps=True),
        pb.Group([pb.TaitEOS('fluid', None, rho0=1., c0=1., gamma=7.)])])],
        names, 3)
    assert [o[0] for o in ops] == ['pair', 'update_nnps', 'eos']


def test_equation_attributes_mirror_reference():
    e = pb.TaitEOS('f', None, rho0=1000.0, c0=10.0, gamma=7.0)
    assert e.no_source and e.sources is None
    assert e.B == 1000.0 * 100.0 / 7.0 and e.gamma1 == 3.0 and e.rho01 == 1e-3
    m = pb.MomentumEquation('f', ['f', 'b'], c0=10.0)
    assert (m.alpha, m.beta, m.gx, m.tensile_correction) == (1.0, 1.0, 0.0, False)
    k = pb.UpdateSmoothingLengthFerrari('f', None, dim=2, hdx=1.3)
    assert k.dim1 == 0.5
    with pytest.raises(ValueError):
        pb.WendlandQuintic(dim=1)
    assert pb.QuinticSpline(dim=3).radius_scale == 3.0
    assert abs(pb.Gaussian(dim=2).fac - 1.0 / np.pi) < 1e-15
    assert abs(pb.CubicSpline(dim=3).fac - 1.0 / np.pi) < 1e-15


def test_dam_break_geometry_counts():
    # _db_geometry.py:284-432 at the example default dx = 0.02, 1 boundary layer:
    # the docstring of dam_break_3d.py quotes the same lattice
    fluid, boundary, obstacle = geo.dam_break_3d_particles(dx=0.05)
    nx = len(np.mgrid[-0.05:3.22 + 0.05 + 0.005:0.05])
    assert fluid.get_number_of_particles() == 24 * 19 * 11
    assert obstacle.get_number_of_particles() > 0
    n_lattice = nx * len(np.mgrid[-0.55:0.55 + 0.005:0.05]) * \
        len(np.mgrid[-0.05:1.05 + 0.005:0.05])
    assert boundary.get_number_of_particles() < n_lattice
    assert np.all(fluid.h == 1.3 * 0.05) and np.all(fluid.m == 1000.0 * 0.05 ** 3)
    assert fluid.x.min() > 0 and fluid.x.max() <= 1.228 and fluid.z.max() <= 0.55
    assert np.all((boundary.x <= 0) | (boundary.x >= 3.22) | (boundary.z <= 0) |
                  (np.abs(boundary.y) >= 0.5))
    # slab-restricted generation gives the same particles
    a = geo.dam_break_3d_particles(dx=0.05, xrange=(-1.0, 1.0))
    b = geo.dam_break_3d_particles(dx=0.05, xrange=(1.0, 9.0))
    for k in range(3):
        assert a[k].get_number_of_particles() + b[k].get_number_of_particles() \
            == [fluid, boundary, obstacle][k].get_number_of_particles()
    # dam_break_2d.py at its default dx: SURVEY.md 8d quotes 2278 + 1660
    f2, b2 = geo.dam_break_2d_particles(dx=0.03)
    assert f2.get_number_of_particles() == 2278
    assert b2.get_number_of_particles() == 1660
    assert np.all(f2.h == 1.3 * 0.03) and np.all(f2.m == 0.03 ** 2 * 1000.0)
    # the reference quirk: h and m do NOT follow --dx
    f3, b3 = geo.dam_break_2d_particles(dx=0.01)
    assert f3.get_number_of_particles() == 20301
    assert b3.get_number_of_particles() == 4852
    assert np.all(f3.h == 1.3 * 0.03)


def test_particle_array_standin():
    pa = pb.get_particle_array_wcsph(name='f', x=np.arange(5.0), h=0.1)
    assert set(['x0', 'rho0', 'arho', 'dt_cfl', 'dt_force', 'gid', 'tag']) <= \
        set(pa.properties)
    assert pa.gid.dtype == np.uint32 and pa.gid[0] == 2 ** 32 - 1
    assert pa.tag.dtype == np.int32
    pa.set_num_real_particles(3)
    assert pa.get_number_of_particles(real=True) == 3
    assert pa.get('x').size == 3 and pa.get('x', only_real_particles=False).size == 5
    pa.resize(8)
    assert pa.x.size == 8 and pa.x[4] == 4.0 and pa.x[7] == 0.0


def test_domain_manager_descriptor():
    # constructor surface of nnps_base.pyx:226-347 (no device needed)
    import pysph_b200 as pb
    dm = pb.DomainManager(xmin=0, xmax=1, ymin=-1, ymax=2, periodic_in_y=True)
    assert dm.is_periodic and not dm.is_mirror
    assert (dm.periodic_in_x, dm.periodic_in_y, dm.periodic_in_z) == (False, True, False)
    assert not pb.DomainManager().is_periodic
    with pytest.raises(ValueError):
        pb.DomainManager(xmin=1, xmax=0)
    dm = pb.DomainManager(xmin=0, xmax=1, mirror_in_x=True, n_layers=3.0)
    assert dm.is_mirror and not dm.is_periodic and dm.n_layers == 3.0
    assert (dm.mirror_in_x, dm.mirror_in_y, dm.mirror_in_z) == (True, False, False)


def test_edac_program_and_scheme():
    """EDACScheme.get_equations (wc/edac.py:776-880, fluids only) -> one fused
    ('tvf', program) op; what the kernels cannot do is refused at setup."""
    from pysph_b200 import _lib as L
    from pysph_b200 import edac, transport_velocity as tv
    from pysph_b200.equations import Group, SummationDensity
    sch = pb.EDACScheme(['f1', 'f2'], [], dim=3, c0=10., nu=0.01, rho0=1., pb=100.,
                        h=0.02, alpha=0.3, gx=1.0, tdamp=2.0)
    groups = sch.get_equations()
    assert [g.real for g in groups] == [False, True]
    assert [type(e).__name__ for e in groups[1].equations][:5] == [
        'MomentumEquationPressureGradient', 'MomentumEquationArtificialViscosity',
        'MomentumEquationViscosity', 'MomentumEquationArtificialStress', 'EDACEquation']
    ops = build_program(groups, ['f1', 'f2'], 3)
    assert [o[0] for o in ops] == ['tvf']
    P = ops[0][1]
    assert (P.passes, P.fluid_mask, P.bql) == (3, 3, 1)
    assert P.eqbits == L.TVF_PGRAD | L.TVF_AV | L.TVF_VISC | L.TVF_ASTRESS | L.TVF_EDAC
    assert (P.pb, P.nu, P.c0, P.alpha, P.gx, P.tdamp) == (100., 0.01, 10., 0.3, 1.0, 2.0)
    assert abs(P.edac_nu - 0.5 * 0.02 * 10. / 8) < 1e-15       # art_nu, wc/edac.py:651-655
    # the groups alone: two ops, not merged across an unrelated group
    ops = build_program([groups[0]], ['f1', 'f2'], 3)
    assert ops[0][1].passes == 1
    ops = build_program([groups[1]], ['f1', 'f2'], 3)
    assert ops[0][1].passes == 2 and ops[0][1].bql == 0
    # refused: basic SummationDensity mixed in, a fluid that is not a source, real=True density
    with pytest.raises(NotImplementedError):
        build_program([Group([tv.SummationDensity('f1', ['f1']),
                              SummationDensity('f1', ['f1'])], real=False)], ['f1'], 2)
    with pytest.raises(NotImplementedError):
        build_program([Group([tv.SummationDensity('f1', ['f1']),
                              tv.SummationDensity('f2', ['f1', 'f2'])], real=False)],
                      ['f1', 'f2'], 2)
    with pytest.raises(NotImplementedError):
        build_program([Group([tv.SummationDensity('f1', ['f1'])], real=True)], ['f1'], 2)
    # solid walls (wc/edac.py:815-822, :840-842): group 1 + the wall equations, the average
    # pressure in a Group of its own, group 2 with the no-slip term -> ONE fused op
    sch = pb.EDACScheme(['f'], ['w1', 'w2'], dim=2, c0=10., nu=0.01, rho0=1., pb=100., h=0.01,
                        gy=-1.0)
    groups = sch.get_equations()
    assert [g.real for g in groups] == [False, True, True]
    assert [type(e).__name__ for e in groups[0].equations] == ['SummationDensity'] + \
        ['SourceNumberDensity', 'VolumeSummation', 'SolidWallPressureBC', 'SetWallVelocity'] * 2
    ops = build_program(groups, ['f', 'w1', 'w2'], 2)
    assert [o[0] for o in ops] == ['tvf']
    P = ops[0][1]
    assert (P.passes, P.fluid_mask, P.solid_mask, P.bql, P.gy) == (7, 1, 6, 0, -1.0)
    assert P.eqbits == L.TVF_PGRAD | L.TVF_VISC | L.TVF_NOSLIP | L.TVF_ASTRESS | L.TVF_EDAC
    assert build_program(groups[:1], ['f', 'w1', 'w2'], 2)[0][1].passes == 1
    assert build_program(groups[:2], ['f', 'w1', 'w2'], 2)[0][1].passes == 5
    # a wall that lacks one of its four equations, wrong sources, the average pressure inside
    # group 1 although there are walls: refused
    with pytest.raises(NotImplementedError):
        build_program([Group(groups[0].equations[:-1], real=False)], ['f', 'w1', 'w2'], 2)
    with pytest.raises(NotImplementedError):
        build_program([Group([tv.SummationDensity('f', ['f', 'w1']),
                              edac.SourceNumberDensity('w1', ['f', 'w1']),
                              tv.VolumeSummation('w1', ['f', 'w1']),
                              edac.SolidWallPressureBC('w1', ['f']),
                              edac.SetWallVelocity('w1', ['f'])], real=False)], ['f', 'w1'], 2)
    with pytest.raises(NotImplementedError):
        build_program([Group(groups[0].equations + [edac.ComputeAveragePressure('f', ['f', 'w1', 'w2'])],
                             real=False)], ['f', 'w1', 'w2'], 2)
    with pytest.raises(NotImplementedError):
        pb.EDACScheme(['f'], [], dim=2, c0=10., nu=0.01, rho0=1., pb=100., h=0.01,
                      inviscid_solids=['wall']).get_equations()
    # the external-flow branch (pb == 0, wc/edac.py:882-971): EDACStep, the number-density
    # MomentumEquation and XSPHCorrection -- names the WCSPH scheme has too; inside an EDAC
    # Group they are the EDAC kernels' equations
    sch = pb.EDACScheme(['f'], ['w1'], dim=2, c0=10., nu=0.01, rho0=1., pb=0.0, h=0.01,
                        alpha=0.2, eps=0.4, clamp_p=True, gy=-1.0, tdamp=0.5)
    assert [type(s_).__name__ for s_ in sch.get_steppers().values()] == ['EDACStep']
    ops = build_program(sch.get_equations(), ['f', 'w1'], 2)
    assert [o[0] for o in ops] == ['tvf']
    P = ops[0][1]
    assert (P.passes, P.fluid_mask, P.solid_mask, P.bql, P.clamp_p) == (3, 1, 2, 0, 1)
    assert P.eqbits == L.TVF_MOM | L.TVF_AV | L.TVF_VISC | L.TVF_NOSLIP | L.TVF_EDAC | L.TVF_XSPH
    assert (P.eps_xsph, P.gy, P.tdamp, P.c0, P.pb) == (0.4, -1.0, 0.5, 10.0, 0.0)
    with pytest.raises(NotImplementedError):     # XSPH over another array than the fluid itself
        g2 = sch.get_equations()[1]
        g2.equations[-1].sources = ['f', 'w1']
        build_program([g2], ['f', 'w1'], 2)
    # the WCSPH Group with the same two names still goes to the pair kernel
    ops = build_program([pb.Group([pb.MomentumEquation('f', ['f'], c0=1.0, alpha=0.1),
                                   pb.XSPHCorrection('f', ['f'])])], ['f'], 2)
    assert ops[0][0] == 'pair'
    pb.PECIntegrator(f=pb.EDACStep())
    # steppers: EDACTVFStep is accepted, unknown ones are not
    pb.PECIntegrator(f1=pb.EDACTVFStep(), f2=pb.EDACTVFStep())
    with pytest.raises(NotImplementedError):
        pb.PECIntegrator(f1=type('EulerStep', (), {})())


def test_taylor_green_geometry():
    # pysph/examples/taylor_green.py:146-166 (dt), :268-297 (lattice, exact solution)
    p = geo.taylor_green_params(50, dim=2)
    assert abs(p['dt'] - min(0.25 * 0.02 / 11.0, 0.125 * 0.02 ** 2 / 0.01, 0.25)) < 1e-15
    pa = geo.taylor_green_particles(50, dim=2)
    assert pa.get_number_of_particles() == 2500
    assert abs(np.sum(pa.m) - 1.0) < 1e-12
    i = 7 * 50 + 3
    assert abs(pa.u[i] + np.cos(2 * np.pi * pa.x[i]) * np.sin(2 * np.pi * pa.y[i])) < 1e-15
    assert abs(pa.p[i] + 0.25 * (np.cos(4 * np.pi * pa.x[i]) + np.cos(4 * np.pi * pa.y[i]))) < 1e-15
    assert set(('uhat', 'V', 'pavg', 'ap', 'p0', 'auhat')) <= set(pa.properties)
    pa3 = geo.taylor_green_particles(8, dim=3)
    assert pa3.get_number_of_particles() == 512 and np.all(pa3.w == 0.0)
    # divergence-free initial field: sum of u over a periodic lattice vanishes
    assert abs(np.sum(pa3.u)) < 1e-10 and abs(np.sum(pa3.v)) < 1e-10


def test_elastic_program_and_scheme():
    """ElasticSolidsScheme.get_equations (solid_mech/basic.py:604-651) -> one fused
    ('solid', program) op carrying the array constants; what the kernels cannot do is
    refused at setup.  (The kernels themselves are not validated on hardware yet.)"""
    from pysph_b200 import solid_mech as sm
    from pysph_b200.equations import Group
    pa = pb.get_particle_array_elastic_dynamics(
        name='ring', x=np.arange(4.) * 0.1, h=0.13, m=1.0, rho=1.2,
        constants=dict(E=1e3, nu=0.3975, rho_ref=1.2, wdeltap=0.5))
    # get_shear_modulus / get_speed_of_sound, solid_mech/basic.py:19-29,77-83
    assert abs(pa.G[0] - 1e3 / (2 * 1.3975)) < 1e-12
    c0 = np.sqrt(1e3 / (3 * (1 - 2 * 0.3975) * 1.2))
    assert abs(pa.c0_ref[0] - c0) < 1e-12 and np.all(pa.cs == c0)
    assert set(('s00', 's220', 'as12', 'r01', 'v21', 'e0')) <= set(pa.properties)
    sch = pb.ElasticSolidsScheme(['ring'], [], dim=2, alpha=1.0, beta=1.5)
    groups = sch.get_equations()
    assert [type(e).__name__ for e in groups[0].equations] == [
        'IsothermalEOS', 'VelocityGradient2D', 'MonaghanArtificialStress']
    assert [type(e).__name__ for e in groups[1].equations] == [
        'ContinuityEquation', 'MomentumEquationWithStress', 'MonaghanArtificialViscosity',
        'HookesDeviatoricStressRate', 'XSPHCorrection']
    ops = build_program(groups, ['ring'], 2, particle_arrays=[pa])
    assert [o[0] for o in ops] == ['solid']
    P = ops[0][1]
    assert (P.passes, P.grad3d, P.elastic_mask) == (3, 0, 1)
    assert (P.eps, P.alpha, P.beta, P.eps_xsph) == (0.3, 1.0, 1.5, 0.5)
    assert (P.rho_ref[0], P.wdeltap[0], P.n[0]) == (1.2, 0.5, 4.0)
    assert abs(P.c0_ref[0] - c0) < 1e-12 and abs(P.G[0] - pa.G[0]) < 1e-12
    assert pb.ElasticSolidsScheme(['ring'], [], dim=3).use_3d_gradient
    with pytest.raises(ValueError):          # constants are needed
        build_program(groups, ['ring'], 2)
    # rigid `solids` (all = solids + elastic_solids, solid_mech/basic.py:613): sources only
    wall = pb.get_particle_array_elastic_dynamics(name='wall', x=np.zeros(2), rho=1.0, m=1.0,
                                                  h=0.1)
    gw = pb.ElasticSolidsScheme(['ring'], ['wall'], dim=2).get_equations()
    assert gw[1].equations[0].sources == ['wall', 'ring']
    assert gw[1].equations[4].sources == ['ring']                # XSPH: own array only
    Pw = build_program(gw, ['ring', 'wall'], 2, particle_arrays=[pa, wall])[0][1]
    assert (Pw.passes, Pw.elastic_mask, Pw.source_mask) == (3, 1, 3)
    assert P.source_mask == 1
    with pytest.raises(NotImplementedError):  # ONE source set for all pair equations
        bad = pb.ElasticSolidsScheme(['ring'], ['wall'], dim=2).get_equations()
        bad[1].equations[0].sources = ['ring']
        build_program(bad, ['ring', 'wall'], 2, particle_arrays=[pa, wall])
    with pytest.raises(NotImplementedError):  # a group 2 without the stress rate
        build_program([groups[0], Group(groups[1].equations[:3])], ['ring'], 2,
                      particle_arrays=[pa])
    pb.EPECIntegrator(ring=pb.SolidMechStep())
    # rings.py:40-78: two rings of the same size approaching each other
    r = geo.rings_particles(dx=0.004)
    assert r.get_number_of_particles() % 2 == 0
    n2 = r.get_number_of_particles() // 2
    assert np.all(r.u[:n2] > 0) and np.all(r.u[n2:] < 0)
    assert abs(abs(r.u[0]) - 0.059 * r.cs[0]) < 1e-9


@pytest.mark.parametrize('extra', [['--dx', '0.07'],
                                   ['--workload', 'rings', '--dx', '0.0025', '--lz', '0.0075'],
                                   ['--workload', 'taylor_green', '--nx', '10']])
def test_bench_reference_arm_contract(extra):
    """`bench.py --impl reference` (the CPU arm the driver runs beside the GPU arm): one JSON
    line with the contract's keys, for every workload, at a size that takes seconds."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, 'bench.py'), '--impl', 'reference',
                          '--steps', '2', '--warmup', '1'] + extra, capture_output=True,
                         text=True, timeout=300, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['unit'] == 'pairs/s' and d['higher_is_better'] is True
    assert d['metric'] == 'particle_pair_interactions_per_s' and d['value'] > 0
    assert d['steps'] == 2 and d['n_gpus'] == 1 and d['ms_per_step'] > 0
    assert d['cpu_baseline']['kind'] == 'port' and d['cpu_baseline']['cores'] >= 1
    assert d['cpu_baseline']['value'] == d['value'] == d['e2e']['value']
    assert d['e2e']['h2d_bytes_per_step'] == 0 and d['e2e']['d2h_bytes_per_step'] == 0
    assert d['config']['pairs_per_step'] > 0 and 'workload' in d['config']


def test_generic_equations_translate_and_compile_with_nvrtc():
    """The generic-equation fallback without a GPU: user bodies -> CUDA C (codegen.py) -> a
    cubin for sm_90a through NVRTC (compiling needs no device).  The same sources run on the
    emulated library in test_library_on_cpu.py and on the GPU in test_gpu_generic.py."""
    import test_gpu_generic as tg
    from pysph_b200 import codegen
    SimpleEquation, MixedTypeEquation, DumbEquation, EqWithTime, KernelSum = tg._equations()
    MyContinuity, MyMomentum, MyXSPH = tg._generic_wcsph()
    names = ['fluid', 'boundary']
    table = codegen.PropertyTable()
    ops = build_program([
        pb.Group([SimpleEquation('fluid', ['fluid']), MixedTypeEquation('fluid', ['fluid', 'boundary']),
                  KernelSum('boundary', ['fluid'])]),
        pb.Group([MyContinuity('boundary', ['fluid']), MyContinuity('fluid', names),
                  MyMomentum('fluid', names, c0=10.0, alpha=0.1, beta=0.0, gx=0.0, gy=-9.81, gz=0.0),
                  MyXSPH('fluid', ['fluid'], eps=0.5)], start_idx=2)],
        names, 3, kernel=pb.QuinticSpline(dim=3), generic=table)
    assert [o[0] for o in ops] == ['generic', 'range', 'generic']
    g1, g2 = ops[0][1], ops[2][1]
    assert table.user == ['wsum']
    # destinations in order of first mention, a kernel each; sources as bit masks
    assert [(k[0], k[1]) for k in g1.kernels] == [('b2g_fluid', 0), ('b2g_boundary', 1)]
    assert g1.kernels[0][5] == 0b11 and g1.kernels[1][5] == 0b01
    assert [(k[0], k[1], k[2], k[3], k[4]) for k in g2.kernels] == \
        [('b2g_boundary', 1, True, True, False), ('b2g_fluid', 0, True, True, True)]
    assert 'x' not in g2.writes and {'arho', 'au', 'dt_cfl', 'ax'} <= g2.writes
    assert 'pow(' not in g2.source and 'b2_grad(2, 3,' in g2.source
    for g in (g1, g2):
        image = codegen.compile_image(g.source)
        assert image[:4] == b'\x7fELF' and len(image) > 4000
    # equations with hand-written kernels never take this path, and a Group that mixes the
    # two kinds is refused
    ops = build_program([pb.ContinuityEquation('fluid', ['fluid'])], names, 3,
                        kernel=pb.CubicSpline(dim=3))
    assert ops[0][0] == 'pair'
    with pytest.raises(NotImplementedError):
        build_program([pb.Group([pb.ContinuityEquation('fluid', ['fluid']),
                                 SimpleEquation('fluid', ['fluid'])])], names, 3,
                      kernel=pb.CubicSpline(dim=3))
    with pytest.raises(NotImplementedError):       # no kernel object, no generated code
        build_program([SimpleEquation('fluid', ['fluid'])], names, 3)
    # the reference's type declarations, several names at once
    ops = build_program([_Declares('fluid', ['fluid'])], names, 3, kernel=pb.CubicSpline(dim=3))
    src = ops[0][1].source
    assert 'long long i = 0;' in src and 'long long j = 0;' in src and 'double acc[3] = {0.0};' in src
    assert codegen.compile_image(src)[:4] == b'\x7fELF'


class _Declares(pb.Equation):
    def loop(self, d_idx, s_idx, d_au, s_m, XIJ):
        i, j = declare('int', 2)
        acc = declare('matrix(3)')
        for i in range(3):
            for j in range(3):
                acc[i] += XIJ[j] * s_m[s_idx]
        d_au[d_idx] += acc[0] + acc[1] + acc[2]
