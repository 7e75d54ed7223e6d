"""Elastic-dynamics kernels (SURVEY.md 8f-2, BASELINE configs[4]): `k_solid_pass1/2` and
`k_stage_solid` against the reference-generated goldens and the oracle, which IS pinned to
the reference (tests/test_oracle_golden.py: test_elastic_dynamics_matches_reference_bodies).
Also run against the host emulation of the whole library (tests/test_library_on_cpu.py)."""
import numpy as np
import pytest

from helpers import load_golden, rel_err
from oracle import oracle as orc

pytestmark = [pytest.mark.gpu,
              pytest.mark.timeout(180)]

SOLID_FIELDS = ['p', 'arho', 'au', 'av', 'aw', 'ax', 'ay', 'az'] + \
    ['v%d%d' % (i, j) for i in range(3) for j in range(3)] + \
    [pre + k for pre in ('r', 'as') for k in ('00', '01', '02', '11', '12', '22')]


def _arrays(case):
    import pysph_b200 as pb
    pas = []
    for name in case['params']['names']:
        a = case['inputs'][name]
        props = dict((k, np.array(v, dtype=float)) for k, v in a.items() if k[0] != '_')
        consts = dict((k, v[0]) for k, v in case['params']['constants'][name].items())
        pa = pb.get_particle_array_elastic_dynamics(name=name, constants=consts, **props)
        pa.set_num_real_particles(a['_n_real'])
        pas.append(pa)
    return pas


@pytest.mark.parametrize('idx', range(6))      # 4, 5: with a rigid `solids` array as a source
def test_elastic_evaluation_matches_reference_bodies(gpu_device, idx):
    import pysph_b200 as pb
    case = load_golden('solid_cases.json')[idx]
    p = case['params']
    pas = _arrays(case)
    kernel = getattr(pb, case['kernel'])(dim=p['dim'])
    sch = pb.ElasticSolidsScheme(p['elastic'], p['solids'], dim=p['dim'], artificial_stress_eps=p['eps'],
                                 xsph_eps=p['eps_xsph'], alpha=p['alpha'], beta=p['beta'],
                                 use_3d_gradient=p.get('grad3d', False))   # 2-D: what the reference scheme emits
    ae = pb.B200AccelerationEval(pas, sch.get_equations(), kernel)
    nn = pb.B200NNPS(p['dim'], pas, backend=ae.backend, kernel=kernel)
    ae.set_nnps(nn)
    ae.compute(0.0, 1e-6)
    ae.backend.pull_all()
    for pa in pas:
        ref = case['outputs'][pa.name]
        nr = ref['_n_real']
        for f in SOLID_FIELDS:
            want = np.array(ref[f])[:nr]
            if pa.name in p['solids']:      # a destination of nothing: what it carried (fp32 on the device)
                assert np.allclose(pa.properties[f][:nr], want, rtol=1e-6, atol=0), (pa.name, f)
                continue
            assert rel_err(pa.properties[f][:nr], want) <= 5e-5, (pa.name, f)
        assert np.all(pa.au[nr:] == 0.0)


def test_solid_mech_step_matches_reference_bodies(gpu_device):
    import pysph_b200 as pb
    g = load_golden('solid_stepper.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        pa = pb.get_particle_array_elastic_dynamics(name='f', **props)
        be = pb.B200Backend([pa])
        be.ctx.call('b200sph_stage_solid', 0, which, g['dt'])
        be.pull_all()
        for k, v in g['outputs'][key].items():
            if k in ('e', 'e0', 'ae'):
                continue                  # not mirrored on the device (no energy equation)
            # accelerations are fp32 on the device: 6e-8 of |a| * dt
            assert np.allclose(pa.properties[k], v, rtol=0, atol=1e-7), (key, k)


def test_rings_steps_vs_oracle(gpu_device):
    """Colliding rings (rings.py) at dx = 0.002 (1.1 k particles), EPEC + SolidMechStep,
    30 fixed steps (the rings touch after ~10) against the oracle."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    dx, dt = 0.002, 1e-7
    pa = geo.rings_particles(dx=dx)
    ref = geo.rings_particles(dx=dx)
    sch = pb.ElasticSolidsScheme(['solid'], [], dim=2)
    s = pb.make_elastic_solver([pa], sch, pb.CubicSpline(dim=2), dt=dt)
    o = orc.ElasticOracleSolver([ref], dict(dim=2, dt=dt, eps=0.3, alpha=1.0, beta=1.0,
                                            eps_xsph=0.5), 'CubicSpline')
    s.initialise()
    o.initialise()
    s.pull()
    for f in ('p', 'au', 'av', 'arho', 'as00', 'as01', 'as11', 'v00', 'v01', 'v10', 'v11'):
        want = ref.properties[f]
        if np.max(np.abs(want)) == 0.0:
            continue
        assert rel_err(pa.properties[f], want) <= 5e-5, f
    for _ in range(30):
        s.step()
        o.step()
    s.pull()
    assert np.max(np.abs(ref.s00)) > 1.0          # the rings are in contact
    for f, tol in (('x', 1e-7), ('y', 1e-7), ('u', 1e-5), ('v', 1e-5), ('rho', 1e-6),
                   ('s00', 1e-4), ('s01', 1e-4), ('s11', 1e-4)):
        want = ref.properties[f]
        scale = max(np.max(np.abs(want)), 1e-12)
        assert np.max(np.abs(pa.properties[f] - want)) <= tol * scale, f


def test_rings_3d_steps_vs_oracle(gpu_device, dx=0.0025, lz=0.0075, steps=12):
    """BASELINE configs[4]'s body at test size: the rings extruded along z
    (geometry.rings_3d_particles), VelocityGradient3D, EPEC + SolidMechStep against the
    oracle; z-symmetry of the tubes is preserved to rounding."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    dt = 1e-7
    pa = geo.rings_3d_particles(dx=dx, lz=lz)
    ref = geo.rings_3d_particles(dx=dx, lz=lz)
    sch = pb.ElasticSolidsScheme(['solid'], [], dim=3)
    s = pb.make_elastic_solver([pa], sch, pb.CubicSpline(dim=3), dt=dt)
    o = orc.ElasticOracleSolver([ref], dict(dim=3, dt=dt, eps=0.3, alpha=1.0, beta=1.0,
                                            eps_xsph=0.5, grad3d=True), 'CubicSpline')
    s.initialise()          # (pair counts are not compared: lattice neighbours at exactly
    o.initialise()          #  2h = 3 dx fall either side of the cut-off in fp32 / fp64; W = 0 there)
    for _ in range(steps):
        s.step()
        o.step()
    s.pull()
    assert np.max(np.abs(ref.s00)) > 1.0
    for f, tol in (('x', 1e-7), ('y', 1e-7), ('z', 1e-7), ('u', 1e-5), ('v', 1e-5),
                   ('w', 1e-5), ('rho', 1e-6), ('s00', 1e-4), ('s01', 1e-4), ('s11', 1e-4),
                   ('s02', 1e-4), ('s12', 1e-4), ('s22', 1e-4)):
        want = ref.properties[f]
        scale = max(np.max(np.abs(want)), 1e-12)
        if f == 'w':
            scale = max(scale, np.max(np.abs(ref.u)))
        if f in ('s02', 's12'):
            scale = max(scale, np.max(np.abs(ref.s00)))
        assert np.max(np.abs(pa.properties[f] - want)) <= tol * scale, f


def _bar_and_wall(dx=0.002):
    """An elastic block (12 x 20 particles) flying at 0.05 c0 into a rigid wall of three
    particle layers (a `solids` array of ElasticSolidsScheme: a source, never stepped)."""
    import pysph_b200 as pb
    ax, ay = dx * (np.arange(12) + 0.5), dx * (np.arange(20) - 9.5)
    x, y = [a.ravel() for a in np.meshgrid(ax + 1.2 * dx, ay, indexing='ij')]
    h = 1.3 * dx
    q = dx / h
    w = (1.0 - 1.5 * q * q * (1.0 - 0.5 * q)) * 10.0 / (7.0 * np.pi) / (h * h)
    consts = dict(wdeltap=w, n=4, rho_ref=1.0, E=1e7, nu=0.3975)
    bar = pb.get_particle_array_elastic_dynamics(name='bar', x=x, y=y, m=dx * dx, rho=1.0, h=h,
                                                 constants=consts)
    bar.u[:] = -0.05 * bar.cs
    bar.v[:] = 0.01 * bar.cs * np.sin(40.0 * y)
    wx, wy = [a.ravel() for a in np.meshgrid(-dx * (np.arange(3) + 0.5),
                                             dx * (np.arange(30) - 14.5), indexing='ij')]
    wall = pb.get_particle_array_elastic_dynamics(name='wall', x=wx, y=wy, m=dx * dx, rho=1.0,
                                                  h=h, constants=consts)
    return [bar, wall]


def test_bar_hits_rigid_wall_vs_oracle(gpu_device):
    """ElasticSolidsScheme(['bar'], ['wall']): 40 EPEC steps against the oracle; the wall is
    a source of every pair equation (it pushes back through the artificial viscosity and
    the stress terms of the bar), stays where it is, and its properties are untouched."""
    import pysph_b200 as pb
    dt = 2e-8
    pas, ref = _bar_and_wall(), _bar_and_wall()
    sch = pb.ElasticSolidsScheme(['bar'], ['wall'], dim=2)
    s = pb.make_elastic_solver(pas, sch, pb.CubicSpline(dim=2), dt=dt)
    o = orc.ElasticOracleSolver(ref, dict(dim=2, dt=dt, eps=0.3, alpha=1.0, beta=1.0,
                                          eps_xsph=0.5, solids=['wall']), 'CubicSpline')
    for _ in range(40):
        s.step()
        o.step()
    s.pull()
    bar, rbar = pas[0], ref[0]
    assert np.max(rbar.au) > 1e3 * np.max(np.abs(rbar.u)) / 1.0        # it is being stopped
    for f, tol in (('x', 1e-7), ('y', 1e-7), ('u', 1e-5), ('v', 1e-5), ('rho', 1e-6),
                   ('s00', 1e-4), ('s01', 1e-4), ('s11', 1e-4)):
        want = rbar.properties[f]
        scale = max(np.max(np.abs(want)), 1e-12)
        assert np.max(np.abs(bar.properties[f] - want)) <= tol * scale, f
    for f in ('x', 'y', 'u', 'rho', 's00', 'p'):
        assert np.array_equal(pas[1].properties[f], ref[1].properties[f]), f


def test_rings_3d_momentum_and_symmetry_at_size(gpu_device, dx=0.0008, lz=0.024, steps=25,
                                                min_particles=150000):
    """Size-independent properties at a size the oracle does not reach in seconds (3-D rings,
    ~200 k particles): the pair forces of MomentumEquationWithStress + artificial viscosity
    are antisymmetric, so total linear momentum stays what it was (zero: the rings approach
    each other with equal speeds) over EPEC steps; the tubes stay mirror symmetric about
    their mid-plane in z and about the contact plane x = spacing."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pa = geo.rings_3d_particles(dx=dx, lz=lz, u_f=0.2)
    n = pa.get_number_of_particles()
    assert n > min_particles
    sch = pb.ElasticSolidsScheme(['solid'], [], dim=3)
    s = pb.make_elastic_solver([pa], sch, pb.CubicSpline(dim=3), dt=2e-8 * dx / 0.0005)
    z0 = pa.z.copy()
    for _ in range(steps):
        s.step()
    s.pull()
    scale = np.sum(pa.m * np.abs(pa.u))
    for k in ('u', 'v', 'w'):
        assert abs(np.sum(pa.m * pa.properties[k])) <= 2e-6 * scale, k
    assert np.max(np.abs(pa.s00)) > 0.0
    # z mirror symmetry: particle (column, layer j) <-> (column, layer nz-1-j)
    nz = int(round(lz / dx))
    g = pa.gid.astype(np.int64)
    order = np.argsort(g)
    col, lay = g[order] // nz, g[order] % nz
    partner = np.argsort(col * nz + (nz - 1 - lay))
    zs, ws, us = pa.z[order], pa.w[order], pa.u[order]
    assert np.max(np.abs((zs - z0[order]) + (zs[partner] - z0[order][partner]))) <= 1e-9 * lz
    assert np.max(np.abs(ws + ws[partner])) <= 1e-5 * np.max(np.abs(us))
    assert np.max(np.abs(us - us[partner])) <= 1e-5 * np.max(np.abs(us))
