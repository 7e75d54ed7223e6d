"""IISPHScheme on the device (csrc/iisph_kernels.cuh, b200sph_iisph_pass, k_stage_iisph) against
the fp64 oracle (tests/iisph_oracle.py), which tests/test_iisph_on_cpu.py pins to the reference's
own bodies.

Tolerances.  The device forms x_ij, r^2, the accept test and every sum in fp64 but the kernel
polynomial in fp32 (sph_kernel<K>, relative error ~1e-7 of its largest gradient), and stores
au, av, aw in the pool's fp32 slots; the relaxed Jacobi iteration carries these errors through
up to 30 sweeps.  One evaluation is compared to 2e-5 of each field's largest magnitude; runs of
tens of steps, in which the differences grow with the motion, to 1e-4 of the particle spacing
for positions and of the largest magnitude for velocities and pressures.  Iteration counts
must be equal at every evaluation: the cases are chosen so that the convergence metric is not
near the tolerance when the iterations stop.
"""
import ctypes as C

import numpy as np
import pytest

import iisph_oracle as orc_iisph


def _iisph_array(name, **props):
    import pysph_b200 as pb
    return pb.get_particle_array_iisph(name=name, **props)


def dam2d(dx=0.1, hdx=1.3):
    """dam_break_2d.py in its IISPH configuration (:118-126, :159-162, :220-237): the 4 x 4 tank
    with two layers, the 1 x 2 column, QuinticSpline, the fluid shifted by dx / 4, adaptive dt
    from 0.125 * 10 * h / c0; h = hdx dx and m = rho0 dx^2"""
    from pysph_b200.geometry import _block_2d, _tank_2d
    rho0, g = 1000.0, 9.81
    h, m = hdx * dx, dx * dx * rho0
    xt, yt = _tank_2d(dx, 4.0, 4.0, 2, [2, 0])
    xf, yf = _block_2d(dx, 1.0, 2.0, [0.5, 1])
    xf, yf = xf + dx + dx / 4, yf + dx
    fluid = _iisph_array('fluid', x=xf, y=yf, h=h, m=m, rho=rho0)
    wall = _iisph_array('boundary', x=xt, y=yt, h=h, m=m, rho=rho0)
    c0 = 10.0 * np.sqrt(2 * g * 2.0)
    return dict(arrays=[fluid, wall], fluids=['fluid'], solids=['boundary'], dim=2, rho0=rho0,
                g=(0.0, -g, 0.0), nu=0.0, kernel='QuinticSpline', dt=0.125 * 10 * h / c0,
                adaptive=True, dx=dx)


def dam3d(dx=0.1, hdx=1.3):
    """dam_break_3d.py's tank (geometry.dam_break_3d_particles) with IISPH arrays (the
    reference's _db_geometry(iisph=True)), CubicSpline, adaptive dt"""
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx, hdx=hdx, nboundary_layers=2)
    arrays = [_iisph_array(pa.name, **dict((k, pa.properties[k].copy()) for k in
                                           ('x', 'y', 'z', 'h', 'm', 'rho', 'gid')))
              for pa in pas]
    c0 = 10.0 * np.sqrt(2.0 * 9.81 * 0.55)
    return dict(arrays=arrays, fluids=['fluid'], solids=['boundary', 'obstacle'], dim=3,
                rho0=1000.0, g=(0.0, 0.0, -9.81), nu=0.0, kernel='CubicSpline',
                dt=0.125 * 10 * hdx * dx / c0, adaptive=True, dx=dx)


def taylor_green(nx=20, dim=2, perturb=0.1):
    """taylor_green.py with IISPHScheme(has_ghosts=True) (:203-206): the periodic unit box,
    QuinticSpline, nu = U L / Re, fixed dt"""
    from pysph_b200 import geometry as geo
    p = geo.taylor_green_params(nx, dim=dim)
    e = geo.taylor_green_particles(nx, dim=dim, perturb=perturb)
    pa = _iisph_array('fluid', **dict((k, e.properties[k].copy()) for k in
                                      ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'gid')))
    return dict(arrays=[pa], fluids=['fluid'], solids=[], dim=dim, rho0=1.0,
                g=(0.0, 0.0, 0.0), nu=p['nu'], kernel='QuinticSpline', dt=5 * p['dt'],
                adaptive=False, dx=p['dx'], periodic=True, has_ghosts=True)


def tg_domain(dim):
    import pysph_b200 as pb
    kw = dict(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, periodic_in_x=True, periodic_in_y=True)
    if dim == 3:
        kw.update(zmin=0.0, zmax=1.0, periodic_in_z=True)
    return pb.DomainManager(**kw)


def scheme(case, **kw):
    import pysph_b200 as pb
    gx, gy, gz = case['g']
    return pb.IISPHScheme(case['fluids'], case['solids'], case['dim'], case['rho0'],
                          nu=case['nu'], gx=gx, gy=gy, gz=gz,
                          has_ghosts=case.get('has_ghosts', False), **kw)


def solver(case, device_dt=True, **kw):
    import pysph_b200 as pb
    dom = tg_domain(case['dim']) if case.get('periodic') else None
    return pb.make_iisph_solver(case['arrays'], scheme(case, **kw),
                                getattr(pb, case['kernel'])(dim=case['dim']), case['dt'],
                                domain=dom, adaptive_timestep=case['adaptive'],
                                device_dt=device_dt)


def oracle_of(case, **kw):
    arrays = dict((pa.name, dict((k, pa.properties[k].astype(float).copy())
                                 for k in pa.properties)) for pa in case['arrays'])
    L = (1.0, 1.0, 1.0 if case['dim'] == 3 else 0.0) if case.get('periodic') else (0.0, 0.0, 0.0)
    return orc_iisph.Solver(arrays, case['fluids'], case['solids'], case['rho0'], case['kernel'],
                            case['dim'], case['dt'], L=L, adaptive=case['adaptive'],
                            nu=case['nu'], g=case['g'], **kw)


# tolerances of a run against the oracle, per field: positions to a fraction of the spacing,
# the rest to a fraction of the field's largest magnitude.  p is the residual rho0 - rho_adv
# divided by aii dt^2 (PressureSolve's post-loop): it amplifies the fp32 differences of the
# kernel values, and of dt (reduced from the pool's fp32 dt_cfl / dt_force), by ~1e3
RUN_TOL = dict(x=1e-4, y=1e-4, z=1e-4, u=1e-4, v=1e-4, w=1e-4, rho=1e-4, p=5e-3)


def compare(s, o, case, names, tol=RUN_TOL):
    s.pull()
    for pa in case['arrays']:
        if pa.name not in names:
            continue
        A = o.arrays[pa.name]
        for k, rel in tol.items():
            got, want = pa.properties[k], A[k]
            scale = case['dx'] if k in 'xyz' else max(float(np.max(np.abs(want))), 1e-30)
            err = float(np.max(np.abs(got - want))) if got.size else 0.0
            assert err <= rel * scale, (pa.name, k, err, scale)


def run_vs_oracle(case, steps, **kw):
    """tens of steps of the device against the oracle, equal iteration counts at every
    evaluation"""
    import pysph_b200 as pb
    o = oracle_of(case, **kw)
    s = solver(case, **kw)
    s.initialise()
    o.initialise()
    its = [pb.last_iterations(s)[0]]
    for _ in range(steps):
        s.step()
        o.step()
        its.append(pb.last_iterations(s)[0])
    assert its == o.iterations, (its, o.iterations)
    compare(s, o, case, case['fluids'])
    return s, o, its


# the cases of the runs against the oracle: (case, scheme keywords, steps).  The dam breaks run
# with tolerance 1e-3, so that the first evaluations iterate more than min_iterations; 'max'
# reaches max_iterations at every evaluation
RUNS = {
    'dam2d': (lambda: dam2d(0.1), dict(tolerance=1e-3), 30),
    'dam3d': (lambda: dam3d(0.12), dict(tolerance=1e-3), 15),
    'tg2': (lambda: taylor_green(24, 2), {}, 30),
    'tg3': (lambda: taylor_green(10, 3), {}, 10),
    'max': (lambda: dam2d(0.1), dict(tolerance=1e-9), 5),
}


def check_run(name, runs=RUNS):
    make, kw, steps = runs[name]
    s, o, its = run_vs_oracle(make(), steps, **kw)
    assert o.margin() > 0.02       # no decision within 2 % of the tolerance
    if name == 'max':
        assert set(its) == {30}
    elif name.startswith('dam'):
        assert max(its) > 2


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(RUNS))
def test_runs_against_the_oracle(name):
    """the 2-D dam break of dam_break_2d.py's IISPH configuration, a 3-D dam break and the
    periodic Taylor-Green vortex of taylor_green.py in 2-D and 3-D, tens of steps each"""
    check_run(name)


def check_one_evaluation(case, rel=2e-5, **kw):
    """one evaluation: every property the scheme writes, and the compression of each
    iteration's end (the device's last)"""
    import pysph_b200 as pb
    o = oracle_of(case, **kw)
    s = solver(case, **kw)
    s.initialise()
    it, hist = orc_iisph.evaluate(o.arrays, case['fluids'], case['solids'], case['rho0'],
                                  case['kernel'], case['dim'], case['dt'], nu=case['nu'],
                                  g=case['g'], L=o.L, **kw)
    got_it, comp = pb.last_iterations(s)
    assert got_it == it, (got_it, it)
    for f in case['fluids']:
        assert abs(comp[f] - hist[-1][f]) <= 1e-5 * max(hist[-1][f], 1e-12), (comp[f], hist[-1][f])
    s.pull()
    for pa in case['arrays']:
        if pa.get_number_of_particles() == 0:
            continue
        A = o.arrays[pa.name]
        names = ('V',) if pa.name in case['solids'] else (
            'rho', 'uadv', 'vadv', 'wadv', 'rho_adv', 'dii0', 'dii1', 'dii2', 'aii', 'p', 'p0',
            'au', 'av', 'aw', 'dt_cfl', 'dt_force', 'compression')
        for k in names:
            got, want = pa.properties[k], A[k]
            scale = max(float(np.max(np.abs(want))), 1e-30)
            assert float(np.max(np.abs(got - want))) <= rel * scale, (pa.name, k)
    return s


@pytest.mark.gpu
@pytest.mark.parametrize('kernel', orc_iisph.KERNELS)
@pytest.mark.parametrize('dim', [2, 3])
def test_one_evaluation_every_kernel(kernel, dim):
    case = dam2d(0.1) if dim == 2 else dam3d(0.15)
    case['kernel'] = kernel
    check_one_evaluation(case, tolerance=1e-3)


def check_host_dt_is_device_dt(case, steps):
    """the solver's device-resident dt (the evaluation reads it on the device) against dt on
    the host: bitwise"""
    import copy
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    out = []
    for c, dev in ((case, True), (c2, False)):
        s = solver(c, device_dt=dev)
        for _ in range(steps):
            s.step()
        s.pull()
        out.append([pa.properties[k].copy() for pa in c['arrays'] for k in ('x', 'y', 'u', 'v', 'p')])
        out.append(s.dt)
    for a, b in zip(out[0], out[2]):
        assert np.array_equal(a, b)
    assert out[1] == out[3]


@pytest.mark.gpu
def test_host_dt_and_device_dt_are_bitwise_equal():
    check_host_dt_is_device_dt(dam2d(0.1), 10)


def check_two_runs_bitwise(case, steps):
    import copy
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    res = []
    for c in (case, c2):
        s = solver(c)
        for _ in range(steps):
            s.step()
        s.pull()
        res.append([pa.properties[k].copy() for pa in c['arrays'] for k in ('x', 'y', 'z', 'u', 'v', 'w', 'p')])
    for a, b in zip(*res):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal():
    check_two_runs_bitwise(dam2d(0.1), 10)


def check_repeat_starts_from_the_steps_pressure(case):
    """An evaluation repeated after a failed deferred drift check starts from the pressure of
    the step (p0), not from the one the first attempt solved: the repeat gives bitwise what one
    evaluation of the same state on fresh lists gives.  Starting from the solved p would
    change the warm start (piter = p / 2) and with it every result."""
    import copy
    import pysph_b200 as pb
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    s = solver(case, device_dt=False)
    for _ in range(3):
        s.step()
    be, nn, ae = s.backend, s.nnps, s.a_eval
    f = case['arrays'][0]
    # an evaluation on fresh lists, then the state of both solvers
    nn.update_domain()
    nn.update()
    ae.compute(0.0, s.dt)
    s.pull()
    for pa, q in zip(case['arrays'], c2['arrays']):
        for k in pa.properties:
            q.properties[k][:] = pa.properties[k]
    # a jump of a smoothing length: the lists are stale, the evaluation is repeated
    shift = f.h[0] * np.random.RandomState(3).uniform(-1, 1, f.x.size)
    for pa in (f, c2['arrays'][0]):
        pa.x[:] += shift
    be.push(0, ['x'])
    p_step = f.p.copy()
    assert np.any(p_step != 0.0)                    # a warm start to restore
    nn.update(deferred=True)
    ae.compute(0.0, s.dt)
    assert nn.confirm() is True
    nn.update()
    ae.compute(0.0, s.dt)
    s2 = solver(c2, device_dt=False)
    s2.nnps.update_domain()
    s2.nnps.update()
    s2.a_eval.compute(0.0, s.dt)
    s.pull()
    s2.pull()
    assert np.array_equal(f.p0, p_step)
    g = c2['arrays'][0]
    for k in ('p', 'au', 'av', 'rho_adv', 'aii'):
        assert np.array_equal(f.properties[k], g.properties[k]), k
    assert pb.last_iterations(s)[0] == pb.last_iterations(s2)[0]


@pytest.mark.gpu
def test_a_repeated_evaluation_starts_from_the_steps_pressure():
    check_repeat_starts_from_the_steps_pressure(dam2d(0.1))


def check_dump_and_restart(case, steps, tmp_path):
    """a run dumped after `steps` and restarted from the file continues bitwise as the
    uninterrupted run does when it evaluates once more at that point: a restart re-evaluates
    before its first step (initial_acceleration, solver.py:454), and an IISPH evaluation
    advances the pressure, the warm start of the next one.  The file carries p in fp64."""
    import copy
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    c3 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    s = solver(case)
    for _ in range(steps):
        s.step()
    # what load_output and the first step after it do (solver.py:616-624, :454)
    s.nnps.update_domain()
    s.nnps.update()
    s.integrator.initial_acceleration(s.t, s.dt)
    for _ in range(steps):
        s.step()
    s.pull()
    a = solver(c2)
    for _ in range(steps):
        a.step()
    fn = a.dump_output(str(tmp_path), 'iisph')
    b = solver(c3)
    b.load_output(fn)
    for _ in range(steps):
        b.step()
    b.pull()
    assert np.any(case['arrays'][0].p != 0.0)      # a warm start to carry
    for pa, q in zip(case['arrays'], c3['arrays']):
        for k in ('x', 'y', 'u', 'v', 'p'):
            assert np.array_equal(pa.properties[k], q.properties[k]), (pa.name, k)


@pytest.mark.gpu
def test_dump_and_restart(tmp_path):
    case = dam2d(0.1)
    case['adaptive'] = False
    check_dump_and_restart(case, 4, tmp_path)


def check_refusals(case):
    import pysph_b200 as pb
    from pysph_b200 import _lib
    s = solver(case)
    s.initialise()
    prog = [op for op in s.a_eval.ops if op[0] == 'iisph'][0][1]
    ctx = s.backend.ctx
    bad = _lib.IisphProgram()
    C.pointer(bad)[0] = prog
    bad.fluid_mask = 0
    with pytest.raises(RuntimeError, match='bad fluid mask'):
        ctx.call('b200sph_iisph_pass', C.byref(bad), None)
    bad.fluid_mask, bad.solid_mask = prog.fluid_mask, prog.fluid_mask
    with pytest.raises(RuntimeError, match='bad solid mask'):
        ctx.call('b200sph_iisph_pass', C.byref(bad), None)
    bad.solid_mask, bad.max_iterations = prog.solid_mask, 0
    with pytest.raises(RuntimeError, match='iterations'):
        ctx.call('b200sph_iisph_pass', C.byref(bad), None)
    with pytest.raises(RuntimeError, match='stage1 only'):
        ctx.call('b200sph_stage_iisph', 0, 2, 0.1)
    with pytest.raises(NotImplementedError, match='IISPHScheme with the slab decomposition'):
        s.set_parallel_manager(object())
    # other integrators refuse IISPHStep; EulerIntegrator refuses other steppers at stage 1
    with pytest.raises(NotImplementedError, match='IISPHStep'):
        pb.EPECIntegrator(fluid=pb.IISPHStep())
    with pytest.raises(NotImplementedError, match='EulerStep'):
        pb.EulerIntegrator(fluid=pb.WCSPHStep()).stage1()


@pytest.mark.gpu
def test_refusals():
    check_refusals(dam2d(0.2))


def check_ghosts_and_1d_refused():
    import pysph_b200 as pb
    x = np.linspace(0, 1, 20)
    pa = _iisph_array('fluid', x=x, h=0.1, m=0.05, rho=1.0)
    with pytest.raises(RuntimeError, match='2-D and 3-D'):
        pb.make_iisph_solver([pa], pb.IISPHScheme(['fluid'], [], 1, 1.0), pb.CubicSpline(dim=1),
                             0.01).initialise()
    pa = _iisph_array('fluid', x=x, y=x, h=0.1, m=0.05, rho=1.0)
    pa.set_num_real_particles(15)
    with pytest.raises(RuntimeError, match='ghost particles'):
        pb.make_iisph_solver([pa], pb.IISPHScheme(['fluid'], [], 2, 1.0), pb.CubicSpline(dim=2),
                             0.01).initialise()


@pytest.mark.gpu
def test_ghosts_and_1d_are_refused():
    check_ghosts_and_1d_refused()


def check_iisph_named_group_outside_the_scheme_is_generic():
    """The scheme's Groups become one op; a Group of IISPH-named equations that does not form
    the scheme goes where it went before: the generic fallback when its equations carry Python
    bodies (as the reference's own do)"""
    from pysph_b200 import codegen
    from pysph_b200.equations import Equation, Group
    from pysph_b200.program import build_program
    import pysph_b200 as pb
    case = dam2d(0.2)
    eqs = scheme(case).get_equations()
    ops = build_program(eqs, ['fluid', 'boundary'], 2)
    assert [op[0] for op in ops] == ['iisph']
    prog = ops[0][1]
    assert (prog.fluid_mask, prog.solid_mask, prog.min_iterations, prog.max_iterations) == (1, 2, 2, 30)
    assert (prog.rho0, prog.gy, prog.omega, prog.tolerance) == (1000.0, -9.81, 0.5, 1e-2)
    # one Group less is not the scheme: NumberDensity (a descriptor without a body) has no kernel
    with pytest.raises(NotImplementedError, match='NumberDensity'):
        build_program(eqs[:-1], ['fluid', 'boundary'], 2)

    class NumberDensity(Equation):           # the reference's body (iisph.py:37-42)
        def initialize(self, d_idx, d_V):
            d_V[d_idx] = 0.0

        def loop(self, d_idx, d_V, WIJ):
            d_V[d_idx] += WIJ
    ops = build_program([Group(equations=[NumberDensity(dest='boundary', sources=['boundary'])])],
                        ['fluid', 'boundary'], 2, kernel=pb.CubicSpline(dim=2),
                        generic=codegen.PropertyTable())
    assert [op[0] for op in ops] == ['generic']


@pytest.mark.gpu
def test_iisph_named_group_outside_the_scheme_is_not_the_scheme():
    check_iisph_named_group_outside_the_scheme_is_generic()


# ---- the fixture made by the reference's own bodies (tests/gen_iisph_golden.py) ----------------
def fixture_solver(c):
    """a solver on the fixture case's real particles (a periodic box for its ghost case)"""
    import pysph_b200 as pb
    arrays = [_iisph_array(name, **dict((k, np.array(v, dtype=float)) for k, v in c['inputs'][name].items()))
              for name in c['fluids'] + c['solids']]
    dom = None
    if c['L']:
        kw = dict(xmin=0.0, xmax=c['L'], ymin=0.0, ymax=c['L'], periodic_in_x=True, periodic_in_y=True)
        if c['dim'] == 3:
            kw.update(zmin=0.0, zmax=c['L'], periodic_in_z=True)
        dom = pb.DomainManager(**kw)
    sch = pb.IISPHScheme(c['fluids'], c['solids'], c['dim'], c['rho0'], nu=c['nu'], gx=c['g'][0],
                         gy=c['g'][1], gz=c['g'][2], tolerance=c['tolerance'],
                         has_ghosts=bool(c['L']))
    s = pb.make_iisph_solver(arrays, sch, getattr(pb, c['kernel'])(dim=c['dim']), c['dt'],
                             domain=dom)
    return s, arrays


# one evaluation against the reference: 2e-5 of each field's largest magnitude (fp32 kernel
# values), the stepped positions to 2e-5 of the largest displacement
FIX_TOL = 2e-5


def check_fixture(c):
    import pysph_b200 as pb
    s, arrays = fixture_solver(c)
    s.initialise()
    it, comp = pb.last_iterations(s)
    assert it == c['iterations'], (c['kernel'], c['dim'], it, c['iterations'])
    for f in c['fluids']:
        want = c['compression'][-1][f]
        assert abs(comp[f] - want) <= 1e-6 * max(want, 1e-9), (f, comp[f], want)
    s.integrator.dt = c['dt']
    s.integrator.stage1()
    s.pull()
    for pa in arrays:
        out = c['outputs'][pa.name]
        for k, v in out.items():
            want = np.array(v)
            got = pa.properties[k[5:] if k.startswith('step_') else k]
            err = float(np.max(np.abs(got - want)))
            if k.startswith('step_') and k[5:] in 'xyz':
                want = want - np.array(c['inputs'][pa.name][k[5:]])   # the displacement
            scale = max(float(np.max(np.abs(want))), 1e-30)
            assert err <= FIX_TOL * scale, (c['kernel'], c['dim'], pa.name, k, err / scale)


@pytest.mark.gpu
def test_fixture():
    from helpers import load_golden
    for c in load_golden('iisph_cases.json'):
        check_fixture(c)


def check_property_ids():
    """the IISPH extension, ids 140 .. 153 (fp64, allocated as a group when one is named):
    push / pull round trips, and the message layout of the halo exchange stays the WCSPH one"""
    import ctypes as C
    import pysph_b200 as pb
    n = 5
    be = pb.B200Backend([pb.get_particle_array_wcsph(name='f', x=np.zeros(n))])
    h, m = C.c_int(), C.c_int()
    for p in range(140, 154):
        v = p + np.arange(n) / 3.0
        be.ctx.call('b200sph_push_f64', 0, p, v.ctypes.data, 0, n)
        out = np.zeros(n)
        be.ctx.call('b200sph_pull_f64', 0, p, out.ctypes.data, 0, n)
        assert np.array_equal(out, v), p
    be.ctx.call('b200sph_halo_layout', C.byref(h), C.byref(m))
    assert (h.value, m.value) == (9, 17)
    for p in (126, 139, 154):
        with pytest.raises(RuntimeError):
            be.ctx.call('b200sph_push_f64', 0, p, np.zeros(n).ctypes.data, 0, n)


@pytest.mark.gpu
def test_property_ids():
    check_property_ids()
