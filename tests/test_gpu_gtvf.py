"""GTVFScheme on the device (csrc/gtvf_kernels.cuh, b200sph_gtvf_pass, k_stage_gtvf) against the
fp64 oracle (tests/gtvf_oracle.py), which tests/test_gtvf_on_cpu.py pins to the reference's own
bodies.

Tolerances.  The device forms x_ij, r^2, the accept test and every sum in fp64 but the kernel
polynomial in fp32 (relative error ~1e-7 of its largest value), and stores arho, au, auhat and a
wall's p in the pool's fp32 slots.  One evaluation is compared to 2e-5 of each field's largest
magnitude; runs of tens of steps to 1e-4 of the particle spacing for positions and of the largest
magnitude for velocities, densities and pressures.
"""
import copy
import ctypes as C

import numpy as np
import pytest

import gtvf_oracle as orc


def dam2d(dx=0.1, hdx=1.3):
    """dam_break_2d.py in its GTVF configuration (:127-132, :163-166): the 4 x 4 tank with 4
    wall layers, the 1 x 2 column shifted by dx / 4, QuinticSpline, dt = 0.125 h / c0,
    pref = B gamma = c0^2 rho0, alpha = nu = 0; the walls' rho0 is 0 (setup_properties)"""
    import pysph_b200 as pb
    from pysph_b200.geometry import _block_2d, _tank_2d
    rho0, g = 1000.0, 9.81
    h, m = hdx * dx, dx * dx * rho0
    xt, yt = _tank_2d(dx, 4.0, 4.0, 4, [2, 0])
    xf, yf = _block_2d(dx, 1.0, 2.0, [0.5, 1])
    xf, yf = xf + dx + dx / 4, yf + dx
    fluid = pb.get_particle_array_gtvf(name='fluid', x=xf, y=yf, h=h, m=m, rho=rho0)
    wall = pb.get_particle_array(name='boundary', x=xt, y=yt, h=h, m=m, rho=rho0)
    c0 = 10.0 * np.sqrt(2 * g * 2.0)
    case = dict(arrays=[fluid, wall], fluids=['fluid'], solids=['boundary'], dim=2, rho0=rho0,
                g=(0.0, -g, 0.0), nu=0.0, alpha=0.0, c0=c0, pref=c0 * c0 * rho0,
                kernel='QuinticSpline', dt=0.125 * h / c0, dx=dx)
    scheme(case).setup_properties(case['arrays'])
    return case


def dam3d(dx=0.1, hdx=1.3):
    """dam_break_3d.py's tank (geometry.dam_break_3d_particles) with GTVF arrays, CubicSpline,
    alpha = 0.1 (the artificial viscosity over the walls too)"""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx, hdx=hdx, nboundary_layers=2)
    arrays = [pb.get_particle_array(name=pa.name, **dict((k, pa.properties[k].copy()) for k in
                                                         ('x', 'y', 'z', 'h', 'm', 'rho', 'gid')))
              for pa in pas]
    c0 = 10.0 * np.sqrt(2.0 * 9.81 * 0.55)
    case = dict(arrays=arrays, fluids=['fluid'], solids=['boundary', 'obstacle'], dim=3,
                rho0=1000.0, g=(0.0, 0.0, -9.81), nu=0.0, alpha=0.1, c0=c0,
                pref=c0 * c0 * 1000.0, kernel='CubicSpline', dt=0.125 * hdx * dx / c0, dx=dx)
    scheme(case).setup_properties(case['arrays'])
    return case


def taylor_green(nx=20, dim=2, perturb=0.1):
    """taylor_green.py with GTVFScheme (:183-184, :211-214): the periodic unit box,
    QuinticSpline, nu = U L / Re, pref = p0 = c0^2 rho0, the example's fixed dt"""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    p = geo.taylor_green_params(nx, dim=dim)
    e = geo.taylor_green_particles(nx, dim=dim, perturb=perturb)
    pa = pb.get_particle_array_gtvf(name='fluid', **dict((k, e.properties[k].copy()) for k in
                                                          ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm',
                                                           'rho', 'gid')))
    c0 = p['c0']
    return dict(arrays=[pa], fluids=['fluid'], solids=[], dim=dim, rho0=1.0, g=(0.0, 0.0, 0.0),
                nu=p['nu'], alpha=0.0, c0=c0, pref=c0 * c0 * 1.0, kernel='QuinticSpline',
                dt=p['dt'], dx=p['dx'], periodic=True)


def tg_domain(dim):
    import pysph_b200 as pb
    kw = dict(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, periodic_in_x=True, periodic_in_y=True)
    if dim == 3:
        kw.update(zmin=0.0, zmax=1.0, periodic_in_z=True)
    return pb.DomainManager(**kw)


def scheme(case):
    import pysph_b200 as pb
    gx, gy, gz = case['g']
    return pb.GTVFScheme(case['fluids'], case['solids'], case['dim'], case['rho0'], case['c0'],
                         case['nu'], None, case['pref'], gx=gx, gy=gy, gz=gz, alpha=case['alpha'])


def solver(case, device_dt=True, **kw):
    import pysph_b200 as pb
    dom = tg_domain(case['dim']) if case.get('periodic') else None
    return pb.make_gtvf_solver(case['arrays'], scheme(case),
                               getattr(pb, case['kernel'])(dim=case['dim']), case['dt'],
                               domain=dom, device_dt=device_dt, **kw)


def oracle_of(case):
    arrays = dict((pa.name, dict((k, pa.properties[k].astype(float).copy())
                                 for k in pa.properties)) for pa in case['arrays'])
    L = (1.0, 1.0, 1.0 if case['dim'] == 3 else 0.0) if case.get('periodic') else (0.0, 0.0, 0.0)
    return orc.Solver(arrays, case['fluids'], case['solids'], case['kernel'], case['dim'],
                      case['dt'], case['rho0'], case['pref'], L=L, c0=case['c0'],
                      alpha=case['alpha'], nu=case['nu'], g=case['g'])


RUN_TOL = dict(x=1e-4, y=1e-4, z=1e-4, u=1e-4, v=1e-4, w=1e-4, rho=1e-4, p=1e-4)


def compare(s, o, case, names, tol=RUN_TOL):
    s.pull()
    for pa in case['arrays']:
        if pa.name not in names:
            continue
        A = o.arrays[pa.name]
        for k, rel in tol.items():
            got, want = pa.properties[k], A[k]
            scale = case['dx'] if k in 'xyz' else max(float(np.max(np.abs(want))), 1e-30)
            if k == 'rho':
                want, got = want - case['rho0'], got - case['rho0']   # its change
                scale = max(float(np.max(np.abs(want))), 1e-30)
            err = float(np.max(np.abs(got - want))) if got.size else 0.0
            assert err <= rel * scale, (pa.name, k, err, scale)


def run_vs_oracle(case, steps):
    o = oracle_of(case)
    s = solver(case)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        s.step()
        o.step()
    compare(s, o, case, case['fluids'])
    return s, o


RUNS = {
    'dam2d': (lambda: dam2d(0.1), 40),
    'dam3d': (lambda: dam3d(0.12), 15),
    'tg2': (lambda: taylor_green(24, 2), 30),
    'tg3': (lambda: taylor_green(10, 3), 10),
}


def check_run(name, runs=RUNS):
    make, steps = runs[name]
    run_vs_oracle(make(), steps)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(RUNS))
def test_runs_against_the_oracle(name):
    """dam_break_2d.py's GTVF configuration, a 3-D dam break with alpha > 0 and the periodic
    Taylor-Green vortex in 2-D and 3-D, tens of steps each"""
    check_run(name)


def check_first_step(case):
    """initial_acceleration runs evaluation 0 only: the first step kicks with the au / auhat the
    arrays were created with"""
    f = case['arrays'][0]
    rs = np.random.RandomState(5)
    for k in ('au', 'av', 'auhat', 'avhat'):
        f.properties[k][:] = rs.uniform(-1, 1, f.x.size)
    au0 = f.au.copy()
    o = oracle_of(case)
    s = solver(case)
    s.initialise()
    s.pull()
    assert np.array_equal(f.au, au0.astype(np.float32).astype(float))
    o.initialise()
    s.step()
    o.step()
    compare(s, o, case, case['fluids'])


@pytest.mark.gpu
def test_first_step_kicks_with_the_arrays_accelerations():
    check_first_step(dam2d(0.1))


def check_host_dt_is_device_dt(case, steps):
    """device-resident dt against dt on the host: bitwise; adaptive_timestep=True keeps dt (the
    arrays have no dt_cfl / dt_force)"""
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    out = []
    for c, dev in ((case, True), (c2, False)):
        s = solver(c, device_dt=dev, adaptive_timestep=True)
        for _ in range(steps):
            s.step()
        s.pull()
        out.append([pa.properties[k].copy() for pa in c['arrays'] for k in ('x', 'y', 'u', 'v', 'rho', 'p')])
        out.append(s.dt)
    for a, b in zip(out[0], out[2]):
        assert np.array_equal(a, b)
    assert out[1] == out[3] == case['dt']


@pytest.mark.gpu
def test_host_dt_and_device_dt_are_bitwise_equal():
    check_host_dt_is_device_dt(dam2d(0.1), 10)


def check_two_runs_bitwise(case, steps):
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    res = []
    for c in (case, c2):
        s = solver(c)
        for _ in range(steps):
            s.step()
        s.pull()
        res.append([pa.properties[k].copy() for pa in c['arrays'] for k in ('x', 'y', 'z', 'u', 'v', 'w', 'rho', 'p')])
    for a, b in zip(*res):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal():
    check_two_runs_bitwise(dam2d(0.1), 10)


def check_repeat_keeps_the_stage_density(case):
    """Evaluation 1 repeated after a failed deferred drift check starts from the density stage 2
    produced (kept in rho0), not from the corrected one the first attempt wrote: the repeat
    gives bitwise what one evaluation of the same state on fresh lists gives"""
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    s = solver(case, device_dt=False)
    for _ in range(3):
        s.step()
    s.pull()
    for pa, q in zip(case['arrays'], c2['arrays']):
        for k in pa.properties:
            q.properties[k][:] = pa.properties[k]
    f = case['arrays'][0]
    shift = f.h[0] * np.random.RandomState(3).uniform(-1, 1, f.x.size)
    for pa in (f, c2['arrays'][0]):
        pa.x[:] += shift
    s.backend.push(0, ['x'])
    nn, ae = s.nnps, s.a_evals[1]
    nn.update(deferred=True)
    ae.compute(0.0, s.dt)
    assert nn.confirm() is True
    nn.update()
    ae.compute(0.0, s.dt)
    s2 = solver(c2, device_dt=False)
    s2.a_evals[1].compute(0.0, s.dt)
    s.pull()
    s2.pull()
    g = c2['arrays'][0]
    for k in ('rho', 'rho0', 'rhodiv', 'p', 'au', 'av', 'auhat', 'avhat', 'p0'):
        assert np.array_equal(f.properties[k], g.properties[k]), k


@pytest.mark.gpu
def test_a_repeated_evaluation_keeps_the_stage_density():
    check_repeat_keeps_the_stage_density(dam2d(0.1))


def check_dump_and_restart(case, steps, tmp_path):
    """A run dumped after `steps` and restarted from the file continues bitwise as the
    uninterrupted run does when, at that point, it does what a restart does: the file holds the
    output arrays, so auhat .. awhat start again from the values the arrays were created with
    (0), and initial_acceleration runs evaluation 0 (solver.py:454)"""
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    c3 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    s = solver(case)
    for _ in range(steps):
        s.step()
    f = case['arrays'][0]
    for k in ('auhat', 'avhat', 'awhat'):
        f.properties[k][:] = 0.0
    s.backend.push(0, ['auhat', 'avhat', 'awhat'])
    s.nnps.update_domain()
    s.nnps.update()
    s.integrator.initial_acceleration(s.t, s.dt)
    for _ in range(steps):
        s.step()
    s.pull()
    a = solver(c2)
    for _ in range(steps):
        a.step()
    fn = a.dump_output(str(tmp_path), 'gtvf')
    b = solver(c3)
    b.load_output(fn)
    for _ in range(steps):
        b.step()
    b.pull()
    for pa, q in zip(case['arrays'], c3['arrays']):
        for k in ('x', 'y', 'u', 'v', 'rho', 'p'):
            assert np.array_equal(pa.properties[k], q.properties[k]), (pa.name, k)


@pytest.mark.gpu
def test_dump_and_restart(tmp_path):
    check_dump_and_restart(dam2d(0.1), 4, tmp_path)


def check_refusals(case):
    import pysph_b200 as pb
    from pysph_b200 import _lib
    s = solver(case)
    s.initialise()
    prog = [op for op in s.a_evals[1].ops if op[0] == 'gtvf'][0][1]
    ctx = s.backend.ctx
    bad = _lib.GtvfProgram()
    C.pointer(bad)[0] = prog
    bad.fluid_mask = 3
    with pytest.raises(RuntimeError, match='bad fluid mask'):
        ctx.call('b200sph_gtvf_pass', C.byref(bad), 1)
    bad.fluid_mask, bad.solid_mask = prog.fluid_mask, prog.fluid_mask
    with pytest.raises(RuntimeError, match='bad solid mask'):
        ctx.call('b200sph_gtvf_pass', C.byref(bad), 1)
    bad.solid_mask, bad.nu = prog.solid_mask, 0.1
    with pytest.raises(RuntimeError, match='nu > 0 with walls'):
        ctx.call('b200sph_gtvf_pass', C.byref(bad), 1)
    with pytest.raises(RuntimeError, match='evaluation must be 0 or 1'):
        ctx.call('b200sph_gtvf_pass', C.byref(prog), 2)
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        ctx.call('b200sph_stage_gtvf', 0, 0, 0.1)
    with pytest.raises(NotImplementedError, match='GTVFScheme with the slab decomposition'):
        s.set_parallel_manager(object())
    # only GTVFIntegrator takes GTVFStep, and it takes nothing else
    with pytest.raises(NotImplementedError, match='GTVFStep'):
        pb.EPECIntegrator(fluid=pb.GTVFStep())
    with pytest.raises(NotImplementedError, match='WCSPHStep'):
        pb.GTVFIntegrator(fluid=pb.WCSPHStep())
    # the set-up refusals: two fluids, nu > 0 with walls, a non-zero asigma
    two = pb.GTVFScheme(['fluid', 'f2'], ['boundary'], 2, 1000.0, 10.0, 0.0, None, 1e5)
    from pysph_b200.program import build_program
    for k in (0, 1):
        with pytest.raises(NotImplementedError, match='2 fluid arrays'):
            build_program(two.get_equations().groups[k], ['fluid', 'f2', 'boundary'], 2)
    visc = pb.GTVFScheme(['fluid'], ['boundary'], 2, 1000.0, 10.0, 0.1, None, 1e5)
    with pytest.raises(NotImplementedError, match='nu > 0 and walls'):
        build_program(visc.get_equations().groups[1], ['fluid', 'boundary'], 2)
    fresh = dam2d(0.3)
    fresh['arrays'][0].asigma[0] = 1.0
    with pytest.raises(NotImplementedError, match='asigma'):
        solver(fresh)


@pytest.mark.gpu
def test_refusals():
    check_refusals(dam2d(0.2))


def check_ghosts_and_1d_refused():
    import pysph_b200 as pb
    x = np.linspace(0, 1, 20)
    sch = pb.GTVFScheme(['fluid'], [], 1, 1.0, 10.0, 0.0, None, 100.0)
    pa = pb.get_particle_array_gtvf(name='fluid', x=x, h=0.1, m=0.05, rho=1.0)
    with pytest.raises(RuntimeError, match='2-D and 3-D'):
        pb.make_gtvf_solver([pa], sch, pb.CubicSpline(dim=1), 0.01).initialise()
    sch.dim = 2
    pa = pb.get_particle_array_gtvf(name='fluid', x=x, y=x, h=0.1, m=0.05, rho=1.0)
    pa.set_num_real_particles(15)
    with pytest.raises(RuntimeError, match='ghost particles'):
        pb.make_gtvf_solver([pa], sch, pb.CubicSpline(dim=2), 0.01).initialise()


@pytest.mark.gpu
def test_ghosts_and_1d_are_refused():
    check_ghosts_and_1d_refused()


def check_translation():
    """each evaluation of the scheme is one op, with or without walls, alpha and nu; the EDAC
    scheme's Groups, which share class names with it, still become EDAC ops"""
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    for solids, kw in ((['w'], dict(alpha=0.1)), ([], dict(nu=0.05)), (['w', 'v'], {})):
        sch = pb.GTVFScheme(['f'], solids, 2, 1000.0, 10.0, kw.get('nu', 0.0), None, 1e5,
                            gy=-9.81, alpha=kw.get('alpha', 0.0))
        ms = sch.get_equations()
        assert isinstance(ms, pb.MultiStageEquations) and len(ms.groups) == 2
        names = ['f', 'w', 'v']
        for k in (0, 1):
            ops = build_program(ms.groups[k], names, 2)
            assert [(op[0], op[2]) for op in ops] == [('gtvf', k)]
            prog = ops[0][1]
            assert prog.fluid_mask == 1
            assert prog.solid_mask == sum(1 << names.index(a) for a in solids)
            if k == 1:
                assert (prog.pref, prog.rho0, prog.gy) == (1e5, 1000.0, -9.81)
                assert (prog.alpha, prog.nu) == (kw.get('alpha', 0.0), kw.get('nu', 0.0))
                assert prog.c0 == (10.0 if kw.get('alpha') else 0.0)
    for ext in (False, True):
        edac = pb.EDACScheme(['f'], ['w'], 2, 10.0, 0.0 if ext else 0.01, 1000.0,
                             pb=0.0 if ext else 1.0, h=0.1)
        ops = build_program(edac.get_equations(), ['f', 'w'], 2)
        assert [op[0] for op in ops] == ['tvf']


@pytest.mark.gpu
def test_translation():
    check_translation()


# ---- the fixture made by the reference's own bodies (tests/gen_gtvf_golden.py) -----------------
def fixture_solver(c):
    import pysph_b200 as pb
    arrays = []
    for name in c['fluids'] + c['solids']:
        props = dict((k, np.array(v, dtype=float)) for k, v in c['inputs'][name].items())
        arrays.append(pb.get_particle_array_gtvf(name=name, **props) if name in c['fluids'] else
                      pb.get_particle_array(name=name, **props))
    sch = pb.GTVFScheme(c['fluids'], c['solids'], c['dim'], c['rho0'], c['c0'], c['nu'], None,
                        c['pref'], gx=c['g'][0], gy=c['g'][1], gz=c['g'][2], alpha=c['alpha'])
    sch.setup_properties(arrays)
    for pa in arrays:                        # (setup_properties adds rho0 etc. as zeros)
        for k, v in c['inputs'][pa.name].items():
            pa.properties[k][:] = v
    dom = None
    if c['L']:
        kw = dict(xmin=0.0, xmax=c['L'], ymin=0.0, ymax=c['L'], periodic_in_x=True, periodic_in_y=True)
        if c['dim'] == 3:
            kw.update(zmin=0.0, zmax=c['L'], periodic_in_z=True)
        dom = pb.DomainManager(**kw)
    s = pb.make_gtvf_solver(arrays, sch, getattr(pb, c['kernel'])(dim=c['dim']), c['dt'],
                            domain=dom)
    return s, arrays


FIX_TOL = 2e-5


def _check_out(arrays, want_all, tag, rel=FIX_TOL, shift=None):
    for pa in arrays:
        for k, v in want_all.get(pa.name, {}).items():
            want = np.array(v, dtype=float)
            got = pa.properties[k].astype(float)
            fin = np.isfinite(want)
            # CorrectDensity's rhodiv is inf where a wall with rho0 = 0 is a neighbour
            assert np.array_equal(np.isfinite(got), fin), (tag, pa.name, k)
            want, got = want[fin], got[fin]
            if shift and k in shift:
                want, got = want - shift[k], got - shift[k]
            scale = max(float(np.max(np.abs(want))), 1e-30) if want.size else 1.0
            err = float(np.max(np.abs(got - want))) if want.size else 0.0
            assert err <= rel * scale, (tag, pa.name, k, err / scale)


def check_fixture(c):
    s, arrays = fixture_solver(c)
    s.a_evals[0].compute(0.0, c['dt'])
    s.pull()
    _check_out(arrays, c['eval0'], (c['kernel'], c['dim'], 0))
    s.a_evals[1].compute(0.0, c['dt'])
    s.pull()
    _check_out(arrays, c['eval1'], (c['kernel'], c['dim'], 1), shift={'rho': c['rho0']})
    if c['steps']:
        s, arrays = fixture_solver(c)
        s.initialise()
        for _ in range(c['steps']):
            s.step()
        s.pull()
        x0 = dict((k, np.array(c['inputs']['fluid'][k])) for k in 'xy')
        want = dict(c['stepped'])
        want['fluid'] = dict((k, (np.array(v) - x0[k]) if k in x0 else v)
                             for k, v in want['fluid'].items())
        for k in 'xy':                       # the displacement
            arrays[0].properties[k] = arrays[0].properties[k] - x0[k]
        _check_out(arrays, want, (c['kernel'], c['dim'], 'steps'), rel=1e-4,
                   shift={'rho': c['rho0']})


@pytest.mark.gpu
def test_fixture():
    from helpers import load_golden
    for c in load_golden('gtvf_cases.json'):
        check_fixture(c)


def check_property_ids():
    """rhodiv and p0 of a GTVF fluid: ids 131 and 132 (fp64, allocated as a group when one is
    named): push / pull round trips; the halo message layout stays the WCSPH one"""
    import pysph_b200 as pb
    n = 5
    be = pb.B200Backend([pb.get_particle_array_wcsph(name='f', x=np.zeros(n))])
    h, m = C.c_int(), C.c_int()
    for p in (131, 132):
        v = p + np.arange(n) / 3.0
        be.ctx.call('b200sph_push_f64', 0, p, v.ctypes.data, 0, n)
        out = np.zeros(n)
        be.ctx.call('b200sph_pull_f64', 0, p, out.ctypes.data, 0, n)
        assert np.array_equal(out, v), p
    be.ctx.call('b200sph_halo_layout', C.byref(h), C.byref(m))
    assert (h.value, m.value) == (9, 17)
    for p in (130, 133):
        with pytest.raises(RuntimeError):
            be.ctx.call('b200sph_push_f64', 0, p, np.zeros(n).ctypes.data, 0, n)
    f = pb.get_particle_array_gtvf(name='f', x=np.zeros(n))
    w = pb.get_particle_array(name='w', x=np.zeros(n))
    pb.GTVFScheme(['f'], ['w'], 2, 1.0, 1.0, 0.0, None, 1.0).setup_properties([f, w])
    be = pb.B200Backend([f, w])
    assert (be.prop_ids[0]['p'], be.prop_ids[0]['rhodiv'], be.prop_ids[0]['p0']) == (30, 131, 132)
    assert (be.prop_ids[1]['ug'], be.prop_ids[1]['p']) == (27, 16) and 'rhodiv' not in be.prop_ids[1]


@pytest.mark.gpu
def test_property_ids():
    check_property_ids()
