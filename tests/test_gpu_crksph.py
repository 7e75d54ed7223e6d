"""CRKSPHScheme on the device (csrc/crksph_kernels.cuh, b200sph_crksph_pass, k_stage_crksph)
against the fp64 oracle (tests/crksph_oracle.py), which tests/test_crksph_on_cpu.py pins to the
reference's own bodies.

Tolerances.  Every property is fp64 on the device and every sum is fp64; the kernel polynomial is
evaluated in fp32 (relative error ~1e-7 of its largest value), and the sums run in list order
rather than the reference's ascending order.  The corrections invert m2, whose conditioning
amplifies that error by a few orders, so one evaluation is compared to 1e-5 of each field's
largest magnitude; runs of tens of steps to 1e-4 of the particle spacing for positions and of the
largest magnitude for velocities, densities, pressures and energies.
"""
import copy
import ctypes as C

import numpy as np
import pytest

import crksph_oracle as orc


def taylor_green(nx=20, dim=2, perturb=0.1, e0=0.0):
    """taylor_green.py with CRKSPHScheme (:207-210, :181-182): the periodic unit box,
    QuinticSpline, nu = U L / Re, p0 = 0 (e = 0: p = 0, driven by viscosity only), the example's
    fixed dt; e0 > 0 gives every particle e = e0 (a pressure field)"""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    p = geo.taylor_green_params(nx, dim=dim)
    src = geo.taylor_green_particles(nx, dim=dim, perturb=perturb)
    pa = pb.get_particle_array_crksph(name='fluid', **dict((k, src.properties[k].copy()) for k in
                                                            ('x', 'y', 'z', 'u', 'v', 'w', 'h',
                                                             'm', 'rho', 'gid')))
    pa.e[:] = e0
    case = dict(arrays=[pa], dim=dim, nu=p['nu'], c0=p['c0'], h0=p['h'], kernel='QuinticSpline',
                dt=p['dt'], dx=p['dx'], g=(0.0, 0.0, 0.0), periodic=True)
    scheme(case).setup_properties(case['arrays'])
    return case


def block(dx=0.1, dim=2, e0=1.0, nu=0.0, g=(0.0, -9.81, 0.0)):
    """a jittered block of fluid with e > 0, gravity and h varying by +-10 %, not periodic"""
    import pysph_b200 as pb
    rs = np.random.RandomState(4)
    n = int(round(1.0 / dx))
    ax = np.arange(n) * dx
    grid = np.meshgrid(*([ax] * dim), indexing='ij')
    pts = [q.ravel() + rs.uniform(-0.1, 0.1, q.size) * dx for q in grid]
    kw = dict(x=pts[0], y=pts[1])
    if dim == 3:
        kw['z'] = pts[2]
    npart = pts[0].size
    pa = pb.get_particle_array_crksph(name='fluid', h=1.2 * dx * (1 + 0.1 * rs.uniform(-1, 1, npart)),
                                      m=dx ** dim, rho=1.0, u=0.3 * rs.uniform(-1, 1, npart),
                                      v=0.3 * rs.uniform(-1, 1, npart), **kw)
    pa.e[:] = e0 * (1 + 0.5 * rs.uniform(-1, 1, npart))
    case = dict(arrays=[pa], dim=dim, nu=nu, c0=10.0, h0=1.2 * dx, kernel='CubicSpline', dt=2e-4,
                dx=dx, g=g)
    scheme(case).setup_properties(case['arrays'])
    return case


def tg_domain(dim):
    import pysph_b200 as pb
    kw = dict(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, periodic_in_x=True, periodic_in_y=True)
    if dim == 3:
        kw.update(zmin=0.0, zmax=1.0, periodic_in_z=True)
    return pb.DomainManager(**kw)


def scheme(case):
    import pysph_b200 as pb
    gx, gy, gz = case['g']
    return pb.CRKSPHScheme(fluids=['fluid'], dim=case['dim'], nu=case['nu'], rho0=1.0,
                           h0=case['h0'], c0=case['c0'], p0=0.0, gx=gx, gy=gy, gz=gz)


def solver(case, device_dt=True, **kw):
    import pysph_b200 as pb
    dom = tg_domain(case['dim']) if case.get('periodic') else None
    return pb.make_crksph_solver(case['arrays'], scheme(case),
                                 getattr(pb, case['kernel'])(dim=case['dim']), case['dt'],
                                 domain=dom, device_dt=device_dt, **kw)


def oracle_of(case):
    pa = case['arrays'][0]
    A = dict((k, pa.properties[k].astype(float).copy()) for k in
             ('x', 'y', 'z', 'u', 'v', 'w', 'u0', 'v0', 'w0', 'h', 'm', 'rho', 'e'))
    L = (1.0, 1.0, 1.0 if case['dim'] == 3 else 0.0) if case.get('periodic') else (0.0, 0.0, 0.0)
    return orc.Solver(A, case['kernel'], case['dim'], case['dt'], L=L, g=case['g'], nu=case['nu'])


RUN_TOL = dict(x=1e-4, y=1e-4, z=1e-4, u=1e-4, v=1e-4, w=1e-4, rho=1e-4, p=1e-4, e=1e-4)


def compare(s, o, case, tol=RUN_TOL):
    s.pull()
    pa = case['arrays'][0]
    for k, rel in tol.items():
        got, want = pa.properties[k], o.A[k]
        scale = case['dx'] if k in 'xyz' else float(np.max(np.abs(want)))
        if k == 'rho':
            got, want = got - 1.0, want - 1.0              # its change
            scale = float(np.max(np.abs(want)))
        if scale == 0.0:
            assert np.array_equal(got, want), k
            continue
        err = float(np.max(np.abs(got - want)))
        assert err <= rel * scale, (k, err, scale)


def run_vs_oracle(case, steps):
    o = oracle_of(case)
    s = solver(case)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        s.step()
        o.step()
    compare(s, o, case)
    return s, o


RUNS = {
    'tg2': (lambda: taylor_green(24, 2), 30),
    'tg3': (lambda: taylor_green(10, 3, e0=1.0), 10),
    'block2': (lambda: block(0.1, 2), 20),
}


def check_run(name, runs=RUNS):
    make, steps = runs[name]
    run_vs_oracle(make(), steps)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(RUNS))
def test_runs_against_the_oracle(name):
    """taylor_green.py's crksph configuration (2-D, periodic, QuinticSpline, e = 0), a 3-D
    periodic Taylor-Green with e > 0 and a 2-D block with gravity, tens of steps each"""
    check_run(name)


def check_first_step(case):
    """initial_acceleration runs evaluation 0: the first step starts from its au, V and ai"""
    o = oracle_of(case)
    s = solver(case)
    s.initialise()
    o.initialise()
    compare(s, o, case, dict(RUN_TOL, au=1e-5, av=1e-5, V=1e-6, ai=1e-5))
    s.step()
    o.step()
    compare(s, o, case)


@pytest.mark.gpu
def test_first_step_is_initial_acceleration():
    check_first_step(block(0.1, 2))


def _snapshot(case):
    return [pa.properties[k].copy() for pa in case['arrays']
            for k in ('x', 'y', 'z', 'u', 'v', 'w', 'rho', 'p', 'e', 'ae', 'gradv')]


def check_host_dt_is_device_dt(case, steps):
    """device-resident dt against dt on the host: bitwise"""
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    out = []
    for c, dev in ((case, True), (c2, False)):
        s = solver(c, device_dt=dev)
        for _ in range(steps):
            s.step()
        s.pull()
        out.append(_snapshot(c))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_host_dt_and_device_dt_are_bitwise_equal():
    check_host_dt_is_device_dt(taylor_green(16, 2, e0=1.0), 10)


def check_two_runs_bitwise(case, steps):
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    res = []
    for c in (case, c2):
        s = solver(c)
        for _ in range(steps):
            s.step()
        s.pull()
        res.append(_snapshot(c))
    for a, b in zip(*res):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal():
    check_two_runs_bitwise(taylor_green(16, 2, e0=1.0), 10)


def check_dump_and_restart(case, steps, tmp_path):
    """A run dumped after `steps` and restarted from the file continues bitwise as the
    uninterrupted run does when, at that point, it does what a restart does: initial_acceleration
    runs evaluation 0 (solver.py:454), which recomputes everything a step reads besides the
    output arrays (x .. w, rho, p, V, e)"""
    c2 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    c3 = dict(case, arrays=[copy.deepcopy(pa) for pa in case['arrays']])
    s = solver(case)
    for _ in range(steps):
        s.step()
    s.nnps.update_domain()
    s.nnps.update()
    s.integrator.initial_acceleration(s.t, s.dt)
    for _ in range(steps):
        s.step()
    s.pull()
    a = solver(c2)
    for _ in range(steps):
        a.step()
    fn = a.dump_output(str(tmp_path), 'crksph')
    b = solver(c3)
    b.load_output(fn)
    for _ in range(steps):
        b.step()
    b.pull()
    for pa, q in zip(case['arrays'], c3['arrays']):
        for k in ('x', 'y', 'u', 'v', 'rho', 'p', 'e'):
            assert np.array_equal(pa.properties[k], q.properties[k]), (pa.name, k)


@pytest.mark.gpu
def test_dump_and_restart(tmp_path):
    check_dump_and_restart(taylor_green(16, 2, e0=1.0), 4, tmp_path)


def check_strided_layout(case):
    """bi, gradai, gradbi and gradv are indexed with stride dim (crksph.py:154-167): a pull
    writes d i + a (d d i + d g + a) at the front of the buffer and leaves the rest as it was"""
    s = solver(case)
    pa = case['arrays'][0]
    d, n = case['dim'], pa.x.size
    for k in ('bi', 'gradai', 'gradbi', 'gradv'):
        pa.properties[k][:] = 7.0
    s.initialise()
    s.pull()
    o = oracle_of(case)
    o.initialise()
    for k, pw in (('bi', 1), ('gradai', 1), ('gradbi', 2), ('gradv', 2)):
        a = pa.properties[k]
        st = d ** pw
        assert np.all(a[st * n:] == 7.0), k
        want = o.A[k][:, :d] if pw == 1 else o.A[k][:, :d, :d]
        got = a[:st * n].reshape(want.shape)
        scale = max(float(np.max(np.abs(want))), 1e-30)
        assert float(np.max(np.abs(got - want))) <= 1e-5 * scale, k
    # a push carries the same layout back: pushed values come back bitwise
    rs = np.random.RandomState(2)
    vals = rs.uniform(-1, 1, d * d * n)
    pa.gradbi[:d * d * n] = vals
    s.backend.push(0, ['gradbi'])
    pa.gradbi[:d * d * n] = 0.0
    s.backend.pull(0, ['gradbi'])
    assert np.array_equal(pa.gradbi[:d * d * n], vals)


@pytest.mark.gpu
def test_strided_layout():
    check_strided_layout(block(0.1, 2))
    check_strided_layout(block(0.25, 3, g=(0.0, 0.0, -9.81)))


def check_reproducing(case, tol):
    """the reproducing property (pysph/sph/tests/test_kernel_corrections.py::test_crksph): after
    the pre-step, interior particles of a perturbed lattice have sum_j V_j W^R_ij = 1 and
    sum_j V_j x_ij W^R_ij = 0, W^R_ij = A_i (1 + B_i . x_ij) W_ij"""
    s = solver(case)
    s.initialise()
    s.pull()
    pa = case['arrays'][0]
    d = case['dim']
    A = dict((k, pa.properties[k].astype(float).copy()) for k in ('x', 'y', 'z', 'h', 'V', 'ai'))
    A['bi'] = np.zeros((pa.x.size, 3))
    A['bi'][:, :d] = pa.bi[:d * pa.x.size].reshape(-1, d)
    i, j, x, r, hij = orc.pairs(A, A, case['kernel'])
    w, _ = orc._wd(case['kernel'], d, x, r, hij)
    wr = A['ai'][i] * (1 + np.einsum('pa,pa->p', A['bi'][i], x)) * w / A['V'][j]
    n = pa.x.size
    s0 = orc._sum(i, n, wr)
    s1 = orc._sum(i, n, wr[:, None] * x)
    lo, hi = [np.min(A[c]) for c in 'xyz'], [np.max(A[c]) for c in 'xyz']
    margin = orc.RADIUS[case['kernel']] * 1.1 * np.max(A['h'])
    inner = np.ones(n, dtype=bool)
    for c, k in zip(range(d), 'xyz'):
        inner &= (A[k] > lo[c] + margin) & (A[k] < hi[c] - margin)
    assert inner.sum() > 0
    assert np.max(np.abs(s0[inner] - 1.0)) < tol
    assert np.max(np.abs(s1[inner])) < tol * case['dx']


@pytest.mark.gpu
def test_reproducing_property():
    """on the device: 1e-6, the kernel polynomial's fp32 error times the corrections' gain"""
    check_reproducing(block(0.05, 2), 1e-6)


def check_momentum_conservation(case, tol):
    """uniform h in a periodic box without gravity: sum_i m_i a_i = 0 to round-off (the
    symmetrised corrected gradient is antisymmetric in i and j)"""
    s = solver(case)
    s.initialise()
    s.pull()
    pa = case['arrays'][0]
    scale = float(np.sum(pa.m * np.sqrt(pa.au ** 2 + pa.av ** 2 + pa.aw ** 2)))
    for k in ('au', 'av', 'aw'):
        assert abs(float(np.sum(pa.m * pa.properties[k]))) <= tol * scale, k


@pytest.mark.gpu
def test_momentum_conservation():
    check_momentum_conservation(taylor_green(16, 2, perturb=0.0, e0=1.0), 1e-12)


def check_refusals(case):
    import pysph_b200 as pb
    from pysph_b200 import _lib
    s = solver(case)
    s.initialise()
    prog = [op for op in s.a_evals[0].ops if op[0] == 'crksph'][0][1]
    ctx = s.backend.ctx
    bad = _lib.CrksphProgram()
    C.pointer(bad)[0] = prog
    bad.fluid_mask = 3
    with pytest.raises(RuntimeError, match='bad fluid mask'):
        ctx.call('b200sph_crksph_pass', C.byref(bad), 0)
    with pytest.raises(RuntimeError, match='evaluation must be 0 or 1'):
        ctx.call('b200sph_crksph_pass', C.byref(prog), 2)
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        ctx.call('b200sph_stage_crksph', 0, 0, 0.1)
    with pytest.raises(NotImplementedError, match='CRKSPHScheme with the slab decomposition'):
        s.set_parallel_manager(object())
    with pytest.raises(NotImplementedError, match='CRKSPHStep'):
        pb.EPECIntegrator(fluid=pb.CRKSPHStep())
    with pytest.raises(NotImplementedError, match='WCSPHStep'):
        pb.CRKSPHIntegrator(fluid=pb.WCSPHStep())
    two = pb.CRKSPHScheme(['fluid', 'f2'], 2, 1.0, 10.0, 0.0, 0.1, 0.0)
    from pysph_b200.program import build_program
    for k in (0, 1):
        with pytest.raises(NotImplementedError, match='2 fluid arrays'):
            build_program(two.get_equations().groups[k], ['fluid', 'f2'], 2)


@pytest.mark.gpu
def test_refusals():
    check_refusals(block(0.2, 2))


def check_ghosts_1d_and_mirror_refused():
    import pysph_b200 as pb
    x = np.linspace(0, 1, 20)
    sch = pb.CRKSPHScheme(['fluid'], 1, 1.0, 10.0, 0.0, 0.1, 0.0)
    pa = pb.get_particle_array_crksph(name='fluid', x=x, h=0.1, m=0.05, rho=1.0)
    with pytest.raises(RuntimeError, match='2-D and 3-D'):
        pb.make_crksph_solver([pa], sch, pb.CubicSpline(dim=1), 0.01).initialise()
    sch.dim = 2
    pa = pb.get_particle_array_crksph(name='fluid', x=x, y=x, h=0.1, m=0.05, rho=1.0)
    pa.set_num_real_particles(15)
    with pytest.raises(RuntimeError, match='ghost particles'):
        pb.make_crksph_solver([pa], sch, pb.CubicSpline(dim=2), 0.01).initialise()
    pa = pb.get_particle_array_crksph(name='fluid', x=x, y=x, h=0.1, m=0.05, rho=1.0)
    dom = pb.DomainManager(xmin=-0.5, xmax=1.5, ymin=-0.5, ymax=1.5, mirror_in_x=True)
    with pytest.raises((RuntimeError, NotImplementedError), match='mirror'):
        pb.make_crksph_solver([pa], sch, pb.CubicSpline(dim=2), 0.01, domain=dom).initialise()


@pytest.mark.gpu
def test_ghosts_1d_and_mirror_are_refused():
    check_ghosts_1d_and_mirror_refused()


def check_translation():
    """each evaluation of the scheme, with or without has_ghosts and nu, is one op; the EDAC and
    WCSPH schemes' Groups, which share class names with it, still take their own routes"""
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    for nu, ghosts, g in ((0.0, False, (0.0, 0.0, 0.0)), (0.05, True, (0.0, -9.81, 0.0))):
        sch = pb.CRKSPHScheme(['f'], 2, 1.0, 10.0, nu, 0.1, 0.0, gx=g[0], gy=g[1], gz=g[2],
                              has_ghosts=ghosts)
        ms = sch.get_equations()
        assert isinstance(ms, pb.MultiStageEquations) and len(ms.groups) == 2
        for k in (0, 1):
            ops = build_program(ms.groups[k], ['w', 'f'], 2)
            assert [(op[0], op[2]) for op in ops] == [('crksph', k)]
            prog = ops[0][1]
            assert prog.fluid_mask == 2 and prog.gamma == 7.0
            if k == 0:
                assert (prog.nu, prog.gy, prog.cl, prog.cq) == (nu, g[1], 2.0, 1.0)
                assert (prog.eta_crit, prog.eta_fold, prog.eta) == (0.3, 0.2, 0.01)
            else:
                # the scheme does not pass its eta_crit to EnergyEquation, whose default is 0.5
                assert (prog.cl_e, prog.cq_e, prog.eta_crit_e, prog.eta_fold_e) == (2.0, 1.0, 0.5, 0.2)
    edac = pb.EDACScheme(['f'], ['w'], 2, 10.0, 0.01, 1000.0, pb=1.0, h=0.1)
    assert [op[0] for op in build_program(edac.get_equations(), ['f', 'w'], 2)] == ['tvf']
    import pysph_b200.crksph as cr
    assert pb.CRKSPHIntegrator.steppers_supported == ('CRKSPHStep',)
    for cls in (pb.PECIntegrator, pb.EPECIntegrator, pb.TVDRK3Integrator, pb.EulerIntegrator,
                pb.GTVFIntegrator):
        assert 'CRKSPHStep' not in cls.steppers_supported
    assert cr.MomentumEquation.__module__ == 'pysph_b200.crksph'


@pytest.mark.gpu
def test_translation():
    check_translation()


# ---- the fixture made by the reference's own bodies (tests/gen_crksph_golden.py) ---------------
def fixture_solver(c):
    import pysph_b200 as pb
    props = dict((k, np.array(v, dtype=float)) for k, v in c['inputs']['fluid'].items())
    pa = pb.get_particle_array_crksph(name='fluid', **props)
    g = c['g']
    sch = pb.CRKSPHScheme(['fluid'], c['dim'], 1.0, 10.0, c['nu'], 0.1, 0.0, gx=g[0], gy=g[1],
                          gz=g[2])
    sch.setup_properties([pa])
    dom = None
    if c['L']:
        kw = dict(xmin=0.0, xmax=c['L'], ymin=0.0, ymax=c['L'], periodic_in_x=True,
                  periodic_in_y=True)
        if c['dim'] == 3:
            kw.update(zmin=0.0, zmax=c['L'], periodic_in_z=True)
        dom = pb.DomainManager(**kw)
    s = pb.make_crksph_solver([pa], sch, getattr(pb, c['kernel'])(dim=c['dim']), c['dt'], domain=dom)
    return s, pa


FIX_TOL = 1e-5


def _check_out(pa, want_all, tag, rel=FIX_TOL, shift=None):
    for k, v in want_all.items():
        want = np.array(v, dtype=float)
        got = pa.properties[k].astype(float)[:want.size]
        if shift and k in shift:
            want, got = want - shift[k], got - shift[k]
        scale = float(np.max(np.abs(want)))
        if scale == 0.0:
            assert np.array_equal(got, want), (tag, k)
            continue
        err = float(np.max(np.abs(got - want)))
        assert err <= rel * scale, (tag, k, err / scale)


def check_fixture(c):
    s, pa = fixture_solver(c)
    s.a_evals[0].compute(0.0, c['dt'])
    s.pull()
    _check_out(pa, c['eval0']['fluid'], (c['kernel'], c['dim'], c['kind'], 0), shift={'rho': 1.0})
    s.a_evals[1].compute(0.0, c['dt'])
    s.pull()
    _check_out(pa, c['eval1']['fluid'], (c['kernel'], c['dim'], c['kind'], 1))
    if c['steps']:
        s, pa = fixture_solver(c)
        s.initialise()
        for _ in range(c['steps']):
            s.step()
        s.pull()
        want = dict(c['stepped']['fluid'])
        x0 = dict((k, np.array(c['inputs']['fluid'][k])) for k in 'xy')
        for k in 'xy':                       # the displacement
            want[k] = np.array(want[k]) - x0[k]
            pa.properties[k] = pa.properties[k] - x0[k]
        _check_out(pa, want, (c['kernel'], c['dim'], 'steps'), rel=1e-4, shift={'rho': 1.0})


@pytest.mark.gpu
def test_fixture():
    from helpers import load_golden
    for c in load_golden('crksph_cases.json'):
        check_fixture(c)


def check_property_ids():
    """the scheme's fp64 group, ids 160 .. 191 (allocated as a group when one is named): push /
    pull round trips; neighbouring ids stay unknown; a CRKSPH fluid's names map to them"""
    import pysph_b200 as pb
    n = 5
    be = pb.B200Backend([pb.get_particle_array_wcsph(name='f', x=np.zeros(n))])
    for p in (160, 167, 168, 174, 183, 191):
        v = p + np.arange(n) / 3.0
        be.ctx.call('b200sph_push_f64', 0, p, v.ctypes.data, 0, n)
        out = np.zeros(n)
        be.ctx.call('b200sph_pull_f64', 0, p, out.ctypes.data, 0, n)
        assert np.array_equal(out, v), p
    for p in (154, 159, 192):
        with pytest.raises(RuntimeError):
            be.ctx.call('b200sph_push_f64', 0, p, np.zeros(n).ctypes.data, 0, n)
    f = pb.get_particle_array_crksph(name='f', x=np.zeros(n))
    be = pb.B200Backend([f])
    ids = be.prop_ids[0]
    assert (ids['p'], ids['e'], ids['ae'], ids['cs'], ids['V'], ids['ai']) == (30, 160, 161, 162, 163, 164)
    assert (ids['au'], ids['av'], ids['aw'], ids['u0']) == (165, 166, 167, 12)
    assert f.bi.size == 3 * n and f.gradbi.size == 9 * n and f.gradv.size == 9 * n


@pytest.mark.gpu
def test_property_ids():
    check_property_ids()
