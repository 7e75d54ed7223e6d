"""The Interpolator on the device: private mode against the reference's own bodies
(interpolator_cases.json), the cases of the reference's pysph/tools/tests/test_interpolator.py
with their known answers and tolerances, a live Interpolator against a private one on the pulled
arrays (dam break under EPEC and TVD-RK3, periodic EDAC Taylor-Green), a run that probes after
every step against one that does not, and the refusals.

The check_* functions take the sizes as arguments: tests/test_interpolator_on_cpu.py runs the
same checks, smaller, on the library emulation.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import load_golden

pytestmark = pytest.mark.gpu

METHODS = ('shepard', 'sph', 'splash', 'splash_norm', 'order1')
# fp32 sums against the fp64 fixture, measured on an H100 80 GB HBM3 (700 W): the four sums
# within 3.4e-7 of the case's largest value, order1 within 5.0e-6 where the fp64 moment matrix
# has a condition number below 1e4 (its solve amplifies the rounding of the fp32 moments by
# that number).  The bounds leave a margin over those.
SUM_TOL, ORDER1_TOL, ORDER1_COND = 2e-6, 1e-4, 1e4


# ---- helpers ---------------------------------------------------------------------------------
def case_arrays(case):
    import pysph_b200 as pb
    pas = []
    for name in ('fluid', 'solid'):
        a = dict((k, np.array(v, dtype=float)) for k, v in case['arrays'][name].items())
        pas.append(pb.get_particle_array(name=name, **a))
    return pas


def case_domain(case):
    import pysph_b200 as pb
    box = case.get('box')
    if box is None:
        return None
    return pb.DomainManager(xmin=box['lo'][0], xmax=box['hi'][0], periodic_in_x=True)


def _grid_2d(n=101, name='fluid'):
    """the reference test's _make_2d_grid"""
    import pysph_b200 as pb
    dx = 2.0 / (n - 1)
    x, y = np.mgrid[-1. + dx / 2:1.:dx, -1. + dx / 2:1.:dx]
    x, y = x.ravel(), y.ravel()
    z = np.zeros_like(x)
    m = np.ones_like(x)
    return pb.get_particle_array(name=name, x=x, y=y, z=z, h=np.ones_like(x) * 2. * dx, m=m,
                                 p=np.sin(x * np.pi), u=np.cos(x * np.pi), rho=m / (dx * dx))


def _domain_2d():
    import pysph_b200 as pb
    return pb.DomainManager(xmin=-1.0, xmax=1.0, ymin=-1.0, ymax=1.0, periodic_in_x=True,
                            periodic_in_y=True)


# ---- 1. private mode against the reference's bodies ------------------------------------------
def check_fixture(idx):
    import pysph_b200 as pb
    from interpolator_oracle import interpolate as oracle
    c = load_golden('interpolator_cases.json')[idx]
    kernel = getattr(pb, c['kernel'])(dim=c['dim'])
    for method in METHODS:
        pas = case_arrays(c)
        P = c['probes']
        ip = pb.Interpolator(pas, kernel=kernel, x=np.array(P['x']), y=np.array(P['y']),
                             z=np.array(P['z']), domain_manager=case_domain(c), method=method)
        want = np.array(c['results'][method])
        if method != 'order1':
            got = ip.interpolate('f')
            scale = np.max(np.abs(want))
            assert np.max(np.abs(got - want)) <= SUM_TOL * scale, (c['kernel'], c['dim'], method, got, want)
            continue
        _, cond, nnb = oracle(c, 'order1')
        for comp in range(4):
            got = ip.interpolate('f', comp)
            w = want[comp::4]
            scale = np.max(np.abs(want.reshape(-1, 4)[cond < ORDER1_COND]))
            good = cond < ORDER1_COND
            assert np.max(np.abs(got[good] - w[good])) <= ORDER1_TOL * scale, (c['kernel'], c['dim'], comp, got, w)
            # gj_solve's early return leaves 0, on the device as in the reference, where the
            # matrix is singular whatever the rounding: no neighbour, or a collinear
            # neighbourhood (one neighbour gives a rank-1 matrix whose pivots are rounding)
            early = np.isinf(cond) & (nnb != 1)
            assert np.all(got[early] == 0.0) and np.all(w[early] == 0.0)


@pytest.mark.parametrize('idx', list(range(15)))
def test_fixture(idx):
    check_fixture(idx)


# ---- 2. the reference's own tests ----------------------------------------------------------------
def check_reference_cases(n=101, num_points=1000):
    import pysph_b200 as pb
    rs = np.random.RandomState(3)
    # test_should_work_on_2d_data
    pa = _grid_2d(n)
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    np.testing.assert_allclose(ip.interpolate('p'), np.sin(ip.x * np.pi), rtol=5e-3)
    np.testing.assert_allclose(ip.interpolate('u'), np.cos(ip.x * np.pi), rtol=5e-3)
    # test_should_work_with_multiple_arrays
    pa1, pa2 = _grid_2d(n), _grid_2d(n, 'solid')
    pa2.p[:] = 4.0
    pa2.u[:] = 0.2
    ip = pb.Interpolator([pa1, pa2], num_points=num_points, domain_manager=_domain_2d())
    np.testing.assert_allclose(ip.interpolate('p'), (np.sin(ip.x * np.pi) + 4.0) * 0.5, rtol=5e-2)
    np.testing.assert_allclose(ip.interpolate('u'), (np.cos(ip.x * np.pi) + 0.2) * 0.5, rtol=5e-2)
    # test_should_work_with_ghost_particles
    pa = _grid_2d(n)
    npart = pa.get_number_of_particles()
    pa.tag[int(npart // 2):] = 1
    pa.set_num_real_particles(int(npart // 2))   # align_particles: the ghosts are already last
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    np.testing.assert_allclose(ip.interpolate('p'), np.sin(ip.x * np.pi), rtol=5e-3)
    np.testing.assert_allclose(ip.interpolate('u'), np.cos(ip.x * np.pi), rtol=5e-3)
    # test_should_work_with_changed_data
    pa = _grid_2d(n)
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    ip.interpolate('p')
    pa.p *= 2.0
    ip.update()
    np.testing.assert_allclose(ip.interpolate('p'), np.sin(ip.x * np.pi) * 2.0, rtol=5e-2)
    # test_should_be_able_to_update_particle_arrays
    pa, pa_new = _grid_2d(n), _grid_2d(n)
    pa_new.p[:] = np.cos(pa_new.x * np.pi)
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    ip.interpolate('p')
    ip.update_particle_arrays([pa_new])
    np.testing.assert_allclose(ip.interpolate('p'), np.cos(ip.x * np.pi), rtol=5e-3)
    # test_should_correctly_update_domain
    pa = _grid_2d(n)
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    ip.interpolate('p')
    ip.set_domain((0.1, 1.0, 0.1, 1.0, 0.0, 0.0), (11, 11, 1))
    np.testing.assert_allclose(ip.interpolate('p'), np.sin(ip.x * np.pi), atol=5e-3)
    # test_should_work_when_arrays_have_different_props
    pa1, pa2 = _grid_2d(n), _grid_2d(n, 'solid')
    pa1.add_property('junk', default=2.0, type='int')
    ip = pb.Interpolator([pa1, pa2], num_points=num_points, domain_manager=_domain_2d())
    junk = ip.interpolate('junk')
    assert np.allclose(junk, np.ones_like(junk) * 1.0)
    # explicit points, with and without z; set_interpolation_points
    pa = _grid_2d(n)
    x, y = rs.random_sample((2, 5, 5))
    ip = pb.Interpolator([pa], x=x, y=y, z=np.zeros_like(x), domain_manager=_domain_2d())
    p = ip.interpolate('p')
    assert p.shape == x.shape
    np.testing.assert_allclose(p, np.sin(ip.x * np.pi), rtol=5e-3)
    ip = pb.Interpolator([pa], x=x, y=y, domain_manager=_domain_2d())
    p = ip.interpolate('p')
    assert p.shape == x.shape
    np.testing.assert_allclose(p, np.sin(ip.x * np.pi), rtol=5e-3)
    ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d())
    x, y = rs.random_sample((2, 5, 5))
    ip.set_interpolation_points(x=x, y=y)
    p = ip.interpolate('p')
    assert p.shape == x.shape
    np.testing.assert_allclose(p, np.sin(ip.x * np.pi), rtol=5e-3)
    # every method on random points; the order1 gradient; the gradient refusals
    for method in METHODS:
        ip = pb.Interpolator([pa], num_points=num_points, domain_manager=_domain_2d(), method=method)
        x, y = rs.random_sample((2, 5, 5))
        ip.set_interpolation_points(x=x, y=y)
        np.testing.assert_allclose(ip.interpolate('p'), np.sin(ip.x * np.pi), rtol=5e-3)
        if method == 'order1':
            np.testing.assert_allclose(ip.interpolate('p', 1), np.pi * np.cos(ip.x * np.pi), rtol=1e-2)
            with pytest.raises(RuntimeError, match='Only 0, 1, 2, 3'):
                ip.interpolate('p', 4)
        else:
            with pytest.raises(RuntimeError, match="use 'order1'"):
                ip.interpolate('p', 1)


def test_reference_cases():
    check_reference_cases()


# ---- 3. live against private ---------------------------------------------------------------------
def _dam_break(dx, integrator):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from test_gpu_tvdrk3 import _solver
    pas = geo.dam_break_3d_particles(dx=dx)
    params = dict(geo.dam_break_3d_params(dx=dx), integrator=integrator)
    return pb, pas, _solver(pas, params)


def _probes():
    """two probes in the fluid column, by the side wall, at the heights of the obstacle probes
    of dam_break_3d.py:118-121"""
    return np.array([0.8245, 0.8245]), np.array([0.471, 0.471]), np.array([0.021, 0.101])


def check_live_vs_private(dx, integrator, steps):
    pb, pas, s = _dam_break(dx, integrator)
    for _ in range(steps):
        s.step()
    x, y, z = _probes()
    live = [pb.Interpolator(pas, x=x, y=y, z=z, method=m) for m in ('shepard', 'order1')]
    live.append(pb.Interpolator(pas, num_points=500))
    got = [ip.interpolate('p') for ip in live] + [live[1].interpolate('p', 3)]
    assert not live[0]._private
    s.pull()
    copies = []
    for pa in pas:
        q = pb.get_particle_array(name=pa.name, **dict((k, v.copy()) for k, v in pa.properties.items()))
        copies.append(q)
    priv = [pb.Interpolator(copies, x=x, y=y, z=z, method=m) for m in ('shepard', 'order1')]
    priv.append(pb.Interpolator(copies, num_points=500))
    # (the default grid comes from the host arrays' bounds: the same points for both)
    priv[2].set_interpolation_points(live[2].x, live[2].y, live[2].z)
    live[2].set_interpolation_points(live[2].x, live[2].y, live[2].z)
    got[2] = live[2].interpolate('p')
    want = [ip.interpolate('p') for ip in priv] + [priv[1].interpolate('p', 3)]
    assert priv[0]._private
    for g, w in zip(got, want):
        scale = max(np.max(np.abs(w)), 1.0)
        assert np.max(np.abs(g - w)) <= 1e-5 * scale, (g, w)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_live_vs_private(integrator):
    check_live_vs_private(0.04, integrator, steps=20)


# ---- 4. probing leaves the run untouched -----------------------------------------------------------
def check_run_untouched(dx, steps):
    results = []
    for probe in (False, True):
        pb, pas, s = _dam_break(dx, 'EPEC')
        if probe:
            x, y, z = _probes()
            ips = [pb.Interpolator(pas, x=x, y=y, z=z, method=m) for m in ('shepard', 'order1')]
            ips += [pb.Interpolator(pas, num_points=300, method=m) for m in ('shepard', 'order1')]
            s.add_post_step_callback(lambda solver: [ip.interpolate('p') for ip in ips])
        for _ in range(steps):
            s.step()
        st = s.backend.stats()
        s.pull()
        results.append((dict((pa.name, dict((k, v.copy()) for k, v in pa.properties.items())) for pa in pas),
                        [st[k] for k in ('full_builds', 'proactive_builds', 'light_updates')]))
    (a, sa), (b, sb) = results
    assert sa == sb
    for name in a:
        for k in a[name]:
            assert np.array_equal(a[name][k], b[name][k]), (name, k)


def test_run_untouched():
    check_run_untouched(0.04, steps=30)


# ---- 5. periodic EDAC ------------------------------------------------------------------------------
def check_periodic_edac(nx, steps):
    import pysph_b200 as pb
    from test_gpu_edac import _tg, _domain, _scheme
    pa, p = _tg(2, nx)
    s = pb.make_edac_solver([pa], _scheme(p, ['fluid']), pb.QuinticSpline(dim=2), dt=p['dt'],
                            domain=_domain(2))
    for _ in range(steps):
        s.step()
    rs = np.random.RandomState(5)
    x, y = rs.uniform(-0.2, 1.2, (2, 40))     # inside and outside the periodic box
    live = pb.Interpolator([pa], x=x, y=y, domain_manager=_domain(2))
    got = live.interpolate('p')
    s.pull()
    q = pb.get_particle_array_edac(name='fluid', **dict((k, v.copy()) for k, v in pa.properties.items()))
    priv = pb.Interpolator([q], x=x, y=y, domain_manager=_domain(2))
    want = priv.interpolate('p')
    assert not live._private and priv._private
    assert np.max(np.abs(got - want)) <= 1e-5 * np.max(np.abs(want)), (got, want)


def test_periodic_edac():
    check_periodic_edac(32, steps=10)


# ---- 6. refusals -----------------------------------------------------------------------------------
def check_refusals():
    import pysph_b200 as pb
    from pysph_b200 import _lib
    pa = _grid_2d(21)
    with pytest.raises(NotImplementedError, match='equations'):
        pb.Interpolator([pa], num_points=100, equations=[object()])
    with pytest.raises(RuntimeError, match='not implemented'):
        pb.Interpolator([pa], num_points=100, method='order2')
    ip = pb.Interpolator([pa], num_points=100, domain_manager=_domain_2d())
    ctx = ip._backend.ctx
    out = np.zeros(400)
    ok = (C.c_int * 8)(*([ip._temp] + [-1] * 7))

    def call(probe=ip._probe, method=0, kernel=3, dim=2, props=ok, mask=1):
        ctx.call('b200sph_interpolate', probe, method, kernel, dim, props, mask, out.ctypes.data)
    call()
    for kw, msg in ((dict(method=5), 'unknown method'), (dict(kernel=4), 'unknown kernel'),
                    (dict(dim=4), 'dim must be'), (dict(mask=2), 'bad array mask'),
                    (dict(mask=0), 'bad array mask'), (dict(probe=99), 'no probe set'),
                    (dict(props=(C.c_int * 8)(*([500] + [-1] * 7))), 'not a floating-point property'),
                    (dict(props=(C.c_int * 8)(*([_lib.USER_PROP0 + 9] + [-1] * 7))), 'not a floating-point property')):
        with pytest.raises(_lib.B200Error, match=msg):
            call(**kw)
    # a probe smoothing length whose reach spans the periodic box
    big = np.array([0.0])
    pid = ctx.call('b200sph_probe_create', 1, big.ctypes.data, big.ctypes.data, big.ctypes.data, 1.0)
    with pytest.raises(_lib.B200Error, match='wraps onto itself'):
        call(probe=pid)
    ctx.call('b200sph_probe_release', pid)
    with pytest.raises(_lib.B200Error, match='no probe set'):
        call(probe=pid)
    with pytest.raises(_lib.B200Error, match='smoothing length'):
        ctx.call('b200sph_probe_create', 1, big.ctypes.data, big.ctypes.data, big.ctypes.data, 0.0)


def test_refusals():
    check_refusals()
