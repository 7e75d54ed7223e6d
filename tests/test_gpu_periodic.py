"""GPU parity tests of periodic domains (SURVEY.md 8f-1): the cell-grid wrap of
the CUDA path against the oracle, which materialises the periodic ghost images
the way the reference does (nnps_base.pyx:699-940 restated in
oracle/oracle.py).  Fixtures follow pysph/base/tests/test_domain_manager.py
(periodic unit box, Gaussian kernel, h = 1.5 dx) and
pysph/tools/tests/test_sph_evaluator.py:36-52."""
import numpy as np
import pytest

from helpers import ACC_FIELDS, rel_err
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _lattice(dim, n, L=1.0, hdx=1.5):
    import pysph_b200 as pb
    dx = L / n
    ax = np.arange(dx / 2, L, dx)
    g = np.meshgrid(*([ax] * dim), indexing='ij')
    xyz = [a.ravel() for a in g] + [np.zeros(n ** dim)] * (3 - dim)
    pa = pb.get_particle_array_wcsph(name='fluid', x=xyz[0], y=xyz[1], z=xyz[2],
                                     h=hdx * dx, m=dx ** dim, rho=1.0)
    pa.gid[:] = np.arange(n ** dim)
    return pa, dx


def _domain(dim, L=1.0):
    import pysph_b200 as pb
    kw = dict(xmin=0.0, xmax=L, periodic_in_x=True)
    if dim > 1:
        kw.update(ymin=0.0, ymax=L, periodic_in_y=True)
    if dim > 2:
        kw.update(zmin=0.0, zmax=L, periodic_in_z=True)
    return pb.DomainManager(**kw)


def _dom_tuple(dm):
    return ([dm.xmin, dm.ymin, dm.zmin], [dm.xmax, dm.ymax, dm.zmax],
            [int(dm.periodic_in_x), int(dm.periodic_in_y), int(dm.periodic_in_z)])


@pytest.mark.parametrize('dim,n', [(1, 20), (2, 10), (3, 5), (3, 12)])
@pytest.mark.parametrize('shift', [0.0, 0.35])
def test_periodic_lattice_density(gpu_device, dim, n, shift):
    """test_domain_manager.py:22-116 / :250-330: on a periodic lattice every
    particle sees the same neighbourhood: sum_j m_j W_ij is uniform and equals
    the oracle's value computed with materialised ghosts.  With shift != 0 the
    particles start outside the box and update_domain wraps them (:172-194)."""
    import pysph_b200 as pb
    pa, dx = _lattice(dim, n)
    for k in ('x', 'y', 'z')[:dim]:
        pa.properties[k] += shift
    dm = _domain(dim)
    kernel = pb.Gaussian(dim=dim)
    ae = pb.B200AccelerationEval(
        [pa], [pb.SummationDensity(dest='fluid', sources=['fluid'])], kernel)
    nn = pb.B200NNPS(dim, [pa], backend=ae.backend, kernel=kernel, domain=dm)
    ae.set_nnps(nn)
    ae.compute(0.0, 0.0)
    ae.backend.pull_all(['rho', 'x', 'y', 'z', 'gid'])
    # wrapped into the box, exactly like _box_wrap_periodic
    q, _ = _lattice(dim, n)
    for k in ('x', 'y', 'z')[:dim]:
        q.properties[k] += shift
    lo, hi, per = _dom_tuple(dm)
    orc.periodic_box_wrap([q], lo, hi, per)
    order = np.argsort(pa.gid)
    for k in ('x', 'y', 'z'):
        assert np.array_equal(pa.properties[k][order], q.properties[k]), k
    g = orc.periodic_ghosts([q], lo, hi, per, 3.0 * 1.5 * dx)
    assert g[0].get_number_of_particles() > n ** dim
    o = orc.Oracle(g, dim, 'Gaussian')
    o.update_domain()
    o.nnps_update()
    o.pair_pass([(orc.EQ_SUMDENS, 0, [0])], real_only=True)
    ref = g[0].rho[:n ** dim]
    assert np.ptp(ref) < 1e-13                      # the fixture's own invariant
    assert abs(ref[0] - 1.0) < 1e-3                 # m / vol, Gaussian cut at 3h
    assert rel_err(pa.rho[order], ref) <= 2e-6
    # neighbour COUNTS match the ghosted search (indices differ: ghosts vs images)
    for i in (0, n ** dim // 2, n ** dim - 1):
        mine = nn.get_nearest_particles(0, 0, int(np.where(pa.gid == i)[0][0]))
        assert len(mine) == len(o.neighbors(0, 0, i))


def test_sph_evaluator_periodic_fixture(gpu_device):
    """pysph/tools/tests/test_sph_evaluator.py:36-52: two arrays, 1-D, domain
    [-dx/2, 1+dx/2] periodic, destination at x = 0 -> rho = 9.0 (2 places)."""
    import pysph_b200 as pb
    x = np.linspace(0, 1, 10)
    dx = x[1] - x[0]
    src = pb.get_particle_array_wcsph(name='src', x=x, m=1.0, h=dx)
    dest = pb.get_particle_array_wcsph(name='dest', x=np.array([0.0]), h=dx)
    dm = pb.DomainManager(xmin=-dx / 2, xmax=1.0 + dx / 2, periodic_in_x=True)
    kernel = pb.Gaussian(dim=1)
    ae = pb.B200AccelerationEval(
        [dest, src], [pb.SummationDensity(dest='dest', sources=['src'])], kernel)
    nn = pb.B200NNPS(1, [dest, src], backend=ae.backend, kernel=kernel, domain=dm)
    ae.set_nnps(nn)
    ae.compute(0.0, 0.0)
    ae.backend.pull_all(['rho'])
    assert abs(dest.rho[0] - 9.0) < 5e-3
    # without the domain the end particle sees half the support
    ae2 = pb.B200AccelerationEval(
        [dest, src], [pb.SummationDensity(dest='dest', sources=['src'])], kernel)
    nn2 = pb.B200NNPS(1, [dest, src], backend=ae2.backend, kernel=kernel)
    ae2.set_nnps(nn2)
    ae2.compute(0.0, 0.0)
    ae2.backend.pull_all(['rho'])
    assert dest.rho[0] < 7.5


def _periodic_case(dim, n, seed=3, tensile=True):
    """tensile=False runs the pair pass on the 32-byte records; beta != 0 then"""
    import pysph_b200 as pb
    pa, dx = _lattice(dim, n, hdx=1.3)
    rs = np.random.RandomState(seed)
    for k in ('x', 'y', 'z')[:dim]:
        pa.properties[k] += 0.25 * dx * rs.uniform(-1, 1, pa.x.size)
    # a smooth periodic velocity field + noise, density perturbation
    pa.u[:] = np.sin(2 * np.pi * pa.x) * np.cos(2 * np.pi * pa.y) + \
        0.05 * rs.normal(size=pa.x.size)
    pa.v[:] = -np.cos(2 * np.pi * pa.x) * np.sin(2 * np.pi * pa.y)
    if dim == 3:
        pa.w[:] = 0.3 * np.sin(2 * np.pi * pa.z)
    rho0 = 1000.0
    pa.rho[:] = rho0 * (1 + 0.01 * rs.uniform(-1, 1, pa.x.size))
    pa.m[:] = rho0 * dx ** dim
    params = dict(fluids=['fluid'], solids=[], dim=dim, rho0=rho0, c0=10.0,
                  h0=1.3 * dx, hdx=1.3, gamma=7.0, alpha=0.1, beta=0.0 if tensile else 0.3,
                  tensile_correction=tensile, dt0=1e-4, cfl=0.3, integrator='EPEC')
    return pa, params


@pytest.mark.parametrize('dim,n,pattern,tensile,zorder', [
    pytest.param(2, 24, (1, 1, 0), True, False, id='2-24-pattern0'),
    pytest.param(3, 10, (1, 1, 1), True, False, id='3-10-pattern1'),
    pytest.param(3, 10, (1, 0, 1), True, False, id='3-10-pattern2'),
    pytest.param(2, 24, (0, 1, 0), True, False, id='2-24-pattern3'),
    pytest.param(2, 24, (1, 1, 0), False, False, id='2-24-pattern0-no_tensile'),
    pytest.param(3, 10, (1, 0, 1), False, False, id='3-10-pattern2-no_tensile'),
    # 3-D n = 9: every axis pattern in row-major order, two of them along the Z-curve
    pytest.param(3, 9, (1, 1, 1), True, False, id='3-9-pattern1'),
    pytest.param(3, 9, (1, 0, 1), True, False, id='3-9-pattern2'),
    pytest.param(3, 9, (0, 1, 0), True, False, id='3-9-pattern3'),
    pytest.param(3, 9, (1, 1, 1), True, True, id='3-9-pattern1-zorder'),
    pytest.param(3, 9, (0, 1, 0), True, True, id='3-9-pattern3-zorder')])
def test_periodic_wcsph_steps_vs_oracle(gpu_device, dim, n, pattern, tensile, zorder):
    periodic_wcsph_steps_vs_oracle(gpu_device, dim, n, pattern, tensile, zorder)


# (test_library_on_cpu.py runs this on the library emulation; tensile is on unless it says not)
def periodic_wcsph_steps_vs_oracle(gpu_device, dim, n, pattern, tensile=True, zorder=False):
    """5 EPEC steps (continuity + momentum + AV + tensile + XSPH + Tait) in a
    box periodic along `pattern`, against the ghost-materialising oracle: the first
    evaluation's pair count, accelerations, dt terms, p and cs, then the state.
    Without the tensile correction every pair pass takes the 32-byte records;
    zorder orders the cell rows along the Z-curve (B200SPH_ZORDER=1)."""
    import pysph_b200 as pb
    pa, params = _periodic_case(dim, n, tensile=tensile)
    ref_pa, _ = _periodic_case(dim, n, tensile=tensile)
    dm = pb.DomainManager(xmin=0, xmax=1, ymin=0, ymax=1, zmin=0,
                          zmax=1 if dim == 3 else 0,
                          periodic_in_x=bool(pattern[0]),
                          periodic_in_y=bool(pattern[1]),
                          periodic_in_z=bool(pattern[2]))
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('B200SPH_ZORDER', '1' if zorder else '0')
        s = pb.make_wcsph_solver([pa], dict(params), pb.CubicSpline(dim=dim), domain=dm)
    o = orc.WCSPHOracleSolver([ref_pa], dict(params), 'CubicSpline',
                              domain=_dom_tuple(dm))
    s.a_eval.count_pairs = True
    s.initialise()
    o.initialise()
    assert s.a_eval.last_pairs == o.pairs_last_eval
    s.a_eval.count_pairs = False
    s.pull()
    r = o.pas[0]
    nr = r.num_real_particles
    order = np.argsort(pa.gid)
    assert np.array_equal(r.gid[:nr], np.arange(nr))
    for k in ACC_FIELDS + ['p', 'cs']:
        ref = r.properties[k][:nr]
        if np.max(np.abs(ref)) == 0.0:
            assert np.max(np.abs(pa.properties[k])) == 0.0
            continue
        assert rel_err(pa.properties[k][order], ref) <= 2e-5, k
    assert abs(s.dt - o.dt) <= 1e-6 * o.dt
    for _ in range(5):
        s.step()
        o.step()
    s.pull()
    r = o.pas[0]
    order = np.argsort(pa.gid)
    for k in ('x', 'y', 'z', 'u', 'v', 'w', 'rho'):
        ref = r.properties[k][:nr]
        scale = max(np.max(np.abs(ref)), 1e-12)
        assert np.max(np.abs(pa.properties[k][order] - ref)) <= 2e-5 * scale, k
    assert abs(s.t - o.t) <= 1e-6 * o.t
    if not tensile:
        st = s.backend.stats()
        assert st['pair_launches_r32'] == st['pair_launches'] > 0, st


def test_periodic_translation_invariance_and_momentum(gpu_device):
    """Size-independent properties at a larger size (48^3 = 110k particles, all
    axes periodic): shifting the initial state by a non-lattice vector shifts the
    result by the same vector, and total momentum is conserved (no boundaries,
    symmetric pair forces) over 20 steps."""
    import pysph_b200 as pb
    dim, n = 3, 48
    sh = np.array([0.3712, 0.62, 0.1234])
    out = []
    for shift in (np.zeros(3), sh):
        pa, params = _periodic_case(dim, n)
        for d, k in enumerate(('x', 'y', 'z')):
            pa.properties[k] += shift[d]
        dm = _domain(3)
        s = pb.make_wcsph_solver([pa], dict(params), pb.CubicSpline(dim=3), domain=dm)
        s.initialise()
        s.pull()
        p0 = np.array([np.sum(pa.m * pa.properties[k]) for k in ('u', 'v', 'w')])
        for _ in range(20):
            s.step()
        s.pull()
        p1 = np.array([np.sum(pa.m * pa.properties[k]) for k in ('u', 'v', 'w')])
        mass = np.sum(pa.m)
        assert np.max(np.abs(p1 - p0)) <= 2e-6 * mass * 1.0     # |u| ~ 1
        st = s.backend.stats()
        assert st['list_builds'] >= 1
        order = np.argsort(pa.gid)
        out.append(dict((k, pa.properties[k][order].copy())
                        for k in ('x', 'y', 'z', 'u', 'v', 'w', 'rho')))
        assert all(out[-1][k].min() >= 0.0 and out[-1][k].max() <= 1.0
                   for k in ('x', 'y', 'z'))
    a, b = out
    for d, k in enumerate(('x', 'y', 'z')):
        diff = (b[k] - a[k] - sh[d] + 0.5) % 1.0 - 0.5       # minimum image
        assert np.max(np.abs(diff)) <= 2e-6, k
    for k in ('u', 'v', 'w'):
        assert np.max(np.abs(b[k] - a[k])) <= 5e-4 * np.max(np.abs(a[k])), k
    assert np.max(np.abs(b['rho'] - a['rho'])) <= 1e-5 * 1000.0


def test_periodic_errors(gpu_device):
    import pysph_b200 as pb
    pa, dx = _lattice(2, 4)                     # L = 1, cell = 2*1.5*0.25 = 0.75
    dm = _domain(2)
    pa2, _ = _lattice(2, 2, hdx=1.5)            # cell = 2*0.75 = 1.5 > L
    kernel = pb.CubicSpline(dim=2)
    be = pb.B200Backend([pa2])
    with pytest.raises(RuntimeError):
        pb.B200NNPS(2, [pa2], backend=be, kernel=kernel, domain=dm)
    with pytest.raises(ValueError):
        pb.DomainManager(xmin=1, xmax=0)

