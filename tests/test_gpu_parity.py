"""GPU parity tests: the CUDA path (through the C-ABI) against the fp64 oracle
and the golden fixtures generated from the reference.

Tolerances (fp32 pair arithmetic on cell-relative coordinates, fp64 state):
every acceleration-like field f is compared as max|f_gpu - f_ref| <= tol *
max|f_ref| with tol = 2e-5 for single evaluations (stated per test); neighbour
SETS must be identical except for fp32 knife-edge pairs, which are counted.
"""
import numpy as np
import pytest

from helpers import (ACC_FIELDS, arrays_from_dict, copy_arrays, load_golden,
                     rel_err, wcsph_params_from_case)
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

TOL_EVAL = 2e-5


def make_solver(pas, params, kernel_name, **kw):
    import pysph_b200 as pb
    kernel = getattr(pb, kernel_name)(dim=params['dim'])
    p = dict((k, v) for k, v in params.items())
    return pb.make_wcsph_solver(pas, p, kernel, **kw)


def scheme_params(p):
    keep = ('fluids', 'solids', 'dim', 'rho0', 'c0', 'h0', 'hdx', 'gamma', 'gx',
            'gy', 'gz', 'alpha', 'beta', 'tensile_correction', 'hg_correction',
            'update_h', 'summation_density', 'dt0', 'n_damp', 'cfl',
            'integrator')
    return dict((k, v) for k, v in p.items() if k in keep)


# ---------------------------------------------------------------------------
def test_kernels_via_two_particle_density(gpu_device):
    """Every kernel/dim: W from SummationDensity on 2 particles vs the values of
    the reference's compiled kernels (tests/golden/kernels.json)."""
    import pysph_b200 as pb
    for entry in load_golden('kernels.json'):
        name, dim = entry['kernel'], entry['dim']
        kernel = getattr(pb, name)(dim=dim)
        for c in entry['cases'][::3]:
            if c['rij'] >= kernel.radius_scale * c['h'] or c['rij'] < 1e-9:
                continue
            x = np.array([c['xij'][0], 0.0])
            y = np.array([c['xij'][1], 0.0])
            z = np.array([c['xij'][2], 0.0])
            pa = pb.get_particle_array_wcsph(name='f', x=x, y=y, z=z,
                                             h=np.full(2, c['h']),
                                             m=np.array([0.0, 1.0]))
            ae = pb.B200AccelerationEval(
                [pa], [pb.SummationDensity(dest='f', sources=['f'])], kernel)
            nn = pb.B200NNPS(dim, [pa], backend=ae.backend, kernel=kernel)
            ae.set_nnps(nn)
            ae.compute(0.0, 0.0)
            ae.backend.pull_all(['rho'])
            scale = entry['fac'] / c['h'] ** dim
            # fp32 arithmetic: relative to the kernel's own magnitude
            assert abs(pa.rho[0] - c['w']) <= 3e-6 * max(scale, abs(c['w'])), \
                (name, dim, c)


def test_density_1d_fixture(gpu_device):
    # pysph/sph/tests/test_acceleration_eval.py:294-303,341,737-741
    import pysph_b200 as pb
    g = load_golden('density_1d.json')
    pa = pb.get_particle_array_wcsph(name='fluid', x=np.array(g['x']),
                                     h=np.array(g['h']), m=np.array(g['m']))
    kernel = pb.CubicSpline(dim=1)
    ae = pb.B200AccelerationEval(
        [pa], [pb.SummationDensity(dest='fluid', sources=['fluid'])], kernel)
    nn = pb.B200NNPS(1, [pa], backend=ae.backend, kernel=kernel)
    ae.set_nnps(nn)
    ae.count_pairs = True
    ae.compute(0.0, 0.1)
    ae.backend.pull_all(['rho'])
    assert [len(nn.get_nearest_particles(0, 0, i)) for i in range(10)] == \
        g['nbr_counts']
    assert ae.last_pairs == sum(g['nbr_counts'])
    assert np.allclose(pa.rho, g['rho'], rtol=2e-6)
    # the reference's own fp32 GPU tolerance for this fixture
    assert np.allclose(pa.rho, [7.357] + [9.0] * 8 + [7.357], atol=1e-2)


@pytest.mark.parametrize('idx', range(6))
def test_wcsph_evaluation_vs_reference_bodies(gpu_device, idx):
    """One AccelerationEval.compute on the golden 3-array cases."""
    case = load_golden('wcsph_cases.json')[idx]
    pas = arrays_from_dict(case['inputs'])
    s = make_solver(pas, scheme_params(wcsph_params_from_case(case)),
                    case['kernel'])
    s.a_eval.count_pairs = True
    s.a_eval.compute(0.0, 0.0)
    s.pull()
    # pair count == oracle pair count (neighbour sets are identical)
    opas = arrays_from_dict(case['inputs'])
    osol = orc.WCSPHOracleSolver(opas, wcsph_params_from_case(case),
                                 case['kernel'])
    assert s.a_eval.last_pairs == osol.evaluate()
    for pa in pas:
        ref = case['outputs'][pa.name]
        nr = ref['_n_real']
        for f in ACC_FIELDS:
            want = np.array(ref[f])[:nr]
            got = pa.properties[f][:nr]
            if np.max(np.abs(want)) == 0.0:
                assert np.max(np.abs(got)) == 0.0, (pa.name, f)
                continue
            assert rel_err(got, want) <= TOL_EVAL, (pa.name, f, rel_err(got, want))
        sd = case['params']['summation_density']
        # with summation density rho itself is an fp32 sum (rel. 2e-7), which the
        # EOS amplifies by gamma = 7 on top of the B*(ratio^7 - 1) cancellation
        B = case['params']['rho0'] * case['params']['c0'] ** 2 / case['params']['gamma']
        assert np.allclose(pa.p, ref['p'], rtol=2e-5 if sd else 1e-6,
                           atol=(2e-5 * B) if sd else 1e-3)
        # (with summation density that atol is wider than TOL_EVAL * max|p|)
        assert rel_err(pa.p, ref['p']) <= TOL_EVAL, (pa.name, 'p', rel_err(pa.p, ref['p']))
        assert np.allclose(pa.cs, ref['cs'], rtol=2e-6)
        assert np.allclose(pa.rho, ref['rho'], rtol=2e-6 if case['params'][
            'summation_density'] else 1e-15)


def _random_arrays(seed=123):
    import pysph_b200 as pb
    rs = np.random.RandomState(seed)
    out = []
    for name, n, hv in (('a', 2048, 0.0), ('b', 1024, 0.0), ('c', 1024, 1.0)):
        x, y, z = (rs.uniform(-1, 1, n) for _ in range(3))
        dx = 2.0 / n ** (1. / 3)
        h = np.full(n, 1.2 * dx) * (1.0 + hv * rs.uniform(0, 1, n))
        out.append(pb.get_particle_array_wcsph(name=name, x=x, y=y, z=z, h=h))
    return out


def test_nnps_equals_brute_force(gpu_device):
    """pysph/base/tests/test_nnps.py:303-474: all (src, dst) pairings, constant
    and variable h, against the fp64 brute force."""
    import pysph_b200 as pb
    pas = _random_arrays()
    kernel = pb.CubicSpline(dim=3)
    nn = pb.B200NNPS(3, pas, kernel=kernel)
    o = orc.Oracle(copy_arrays(pas), 3, 'CubicSpline')
    g = nn
    og = None
    o.update_domain()
    o.nnps_update()
    og = o.grid()
    # the grid follows the reference exactly (fp64 on the host)
    assert g.cell_size == og['cell_size']
    assert np.array_equal(g.ncells_per_dim, og['ncells'])
    assert np.allclose(g.xmin, og['xmin'], rtol=0, atol=0)
    rs = np.random.RandomState(0)
    mismatched = 0
    total = 0
    for dst in range(3):
        for src in range(3):
            n = pas[dst].get_number_of_particles()
            for i in rs.randint(0, n, 40):
                a = nn.get_nearest_particles(src, dst, i)
                b = np.sort(o.brute_neighbors(dst, src, i))
                total += len(b)
                mismatched += len(np.setxor1d(a, b))
    # fp32 knife-edge pairs: |r^2 - (kh)^2| within fp32 rounding
    assert mismatched <= 2, (mismatched, total)


def test_nnps_corner_cases(gpu_device):
    import pysph_b200 as pb
    # test_nnps.py:1250-1391
    rs = np.random.RandomState(1)
    n = 2 ** 14
    pb_ = pb.get_particle_array_wcsph(name='b', x=rs.uniform(0, 0.1, n),
                                      y=rs.uniform(0, 0.1, n),
                                      z=rs.uniform(0, 0.1, n), h=np.ones(n))
    nn = pb.B200NNPS(3, [pb_], kernel=pb.CubicSpline(dim=3))
    assert len(nn.get_nearest_particles(0, 0, 5)) == n
    # degenerate dimension: only y varies
    pc = pb.get_particle_array_wcsph(name='c', x=np.zeros(2),
                                     y=np.array([0.0, 0.5]), z=np.zeros(2),
                                     h=np.ones(2))
    for dim in (2, 3):
        nn = pb.B200NNPS(dim, [pc], kernel=pb.CubicSpline(dim=dim))
        assert list(nn.get_nearest_particles(0, 0, 0)) == [0, 1]
    # too many cells -> RuntimeError like linked_list_nnps.pyx:336-343
    pd = pb.get_particle_array_wcsph(name='d', x=np.array([0.0, 1e6]),
                                     y=np.array([0.0, 1e6]),
                                     z=np.array([0.0, 1e6]), h=np.full(2, 0.5))
    with pytest.raises(RuntimeError):
        pb.B200NNPS(3, [pd], kernel=pb.CubicSpline(dim=3))
    # empty + tiny arrays
    pe = pb.get_particle_array_wcsph(name='e', x=np.zeros(0))
    pf = pb.get_particle_array_wcsph(name='f', x=np.array([0.25]), h=np.ones(1))
    nn = pb.B200NNPS(1, [pe, pf], kernel=pb.CubicSpline(dim=1))
    assert list(nn.get_nearest_particles(1, 1, 0)) == [0]
    assert len(nn.get_nearest_particles(0, 1, 0)) == 0


def test_steppers_and_eos_vs_reference_bodies(gpu_device):
    import ctypes as C
    import pysph_b200 as pb
    g = load_golden('steppers.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        pa = pb.get_particle_array_wcsph(name='f', **props)
        be = pb.B200Backend([pa])
        be.ctx.call('b200sph_stage', -1, which, g['dt'])
        be.pull_all()
        for k, v in g['outputs'][key].items():
            # accelerations are fp32 on the device, the state is fp64
            assert np.allclose(pa.properties[k], v, rtol=1e-6, atol=1e-7), (key, k)
    e = load_golden('eos.json')
    for name, hg in (('TaitEOS', 0), ('TaitEOSHGCorrection', 1)):
        d = e[name]
        pa = pb.get_particle_array_wcsph(name='f', x=np.zeros(len(d['rho_in'])),
                                         rho=np.array(d['rho_in']))
        be = pb.B200Backend([pa])
        be.ctx.call('b200sph_eos', 0, hg, d['rho0'], d['c0'], d['gamma'],
                    d['p0'], 0)
        be.pull_all()
        assert np.array_equal(pa.rho, d['rho_out'])
        assert np.allclose(pa.p, d['p'], rtol=1e-6, atol=1e-3)
        assert np.allclose(pa.cs, d['cs'], rtol=1e-6)
    d = e['UpdateSmoothingLengthFerrari']
    pa = pb.get_particle_array_wcsph(name='f', x=np.zeros(len(d['rho'])),
                                     rho=np.array(d['rho']), m=np.array(d['m']))
    be = pb.B200Backend([pa])
    be.ctx.call('b200sph_ferrari_h', 0, d['hdx'], d['dim'], 0)
    be.pull_all()
    assert np.allclose(pa.h, d['h'], rtol=1e-14)


def _compare_state(pas, opas, tol_pos, tol_vel, tol_rho, h0, c0, rho0):
    for pa, oa in zip(pas, opas):
        nr = oa.num_real_particles
        for f in ('x', 'y', 'z'):
            assert np.max(np.abs(pa.properties[f][:nr] - oa.properties[f][:nr])) \
                <= tol_pos * h0, (pa.name, f)
        for f in ('u', 'v', 'w'):
            assert np.max(np.abs(pa.properties[f][:nr] - oa.properties[f][:nr])) \
                <= tol_vel * c0, (pa.name, f)
        assert np.max(np.abs(pa.rho[:nr] - oa.rho[:nr])) <= tol_rho * rho0, pa.name


def test_dam_break_3d_small_eval_and_steps(gpu_device):
    """Config 2 at reduced resolution (dx = 0.05: ~5 k fluid): one evaluation
    and then 20 adaptive EPEC steps against the oracle."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    dx = 0.05
    pas = geo.dam_break_3d_particles(dx=dx)
    params = geo.dam_break_3d_params(dx)
    opas = copy_arrays(pas)
    s = make_solver(pas, scheme_params(params), 'CubicSpline')
    o = orc.WCSPHOracleSolver(opas, params, 'CubicSpline', threads=4)
    s.a_eval.count_pairs = True
    s.initialise()
    o.initialise()
    assert s.a_eval.last_pairs == o.pairs_last_eval
    assert abs(s.dt - o.dt) <= 1e-6 * o.dt
    s.pull()
    for pa, oa in zip(pas, opas):
        nr = oa.num_real_particles
        for f in ACC_FIELDS:
            want = oa.properties[f][:nr]
            got = pa.properties[f][:nr]
            scale = max(np.max(np.abs(want)), 1e-30)
            if f in ('au', 'av', 'aw'):
                scale = max(scale, 9.81)
            assert np.max(np.abs(got - want)) <= TOL_EVAL * scale, (pa.name, f)
    for _ in range(20):
        s.step()
        o.step()
    s.pull()
    assert abs(s.t - o.t) <= 1e-5 * o.t
    _compare_state(pas, opas, tol_pos=1e-6, tol_vel=1e-6, tol_rho=1e-7,
                   h0=params['h0'], c0=params['c0'], rho0=params['rho0'])


def test_dam_break_2d_gate(gpu_device):
    """Config 1 (the reference correctness gate): 2D dam break, WendlandQuintic,
    PEC, update_h, HG correction -- default dx = 0.03, 25 steps."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_2d_particles(dx=0.03)
    params = geo.dam_break_2d_params(dx=0.03)
    opas = copy_arrays(pas)
    s = make_solver(pas, scheme_params(params), 'WendlandQuintic')
    o = orc.WCSPHOracleSolver(opas, params, 'WendlandQuintic', threads=4)
    for _ in range(25):
        s.step()
        o.step()
    s.pull()
    assert abs(s.t - o.t) <= 1e-5 * o.t
    _compare_state(pas, opas, tol_pos=1e-6, tol_vel=1e-6, tol_rho=1e-7,
                   h0=params['h0'], c0=params['c0'], rho0=params['rho0'])
    assert np.allclose(pas[0].h, opas[0].h, rtol=1e-7)


def test_push_pull_roundtrip_and_errors(gpu_device):
    import pysph_b200 as pb
    from pysph_b200._lib import B200Error
    rs = np.random.RandomState(5)
    n = 1000
    pa = pb.get_particle_array_wcsph(name='f', x=rs.normal(size=n),
                                     y=rs.normal(size=n), u=rs.normal(size=n),
                                     rho=rs.uniform(900, 1100, n),
                                     h=np.full(n, 0.1))
    pa.gid[:] = np.arange(n)
    ref = dict((k, v.copy()) for k, v in pa.properties.items())
    be = pb.B200Backend([pa])
    for k in pa.properties:
        pa.properties[k][:] = 0
    be.pull_all()
    for k in ('x', 'y', 'u', 'rho', 'h', 'gid', 'tag'):
        assert np.array_equal(pa.properties[k], ref[k]), k   # fp64 state is exact
    with pytest.raises(B200Error):
        be.ctx.call('b200sph_push_f64', 0, 0, pa.x.ctypes.data, 0, n + 1)
    with pytest.raises(B200Error):
        be.ctx.call('b200sph_push_f64', 3, 0, pa.x.ctypes.data, 0, 1)
    # evaluating before a neighbour build is an error, not a silent stale result
    ae = pb.B200AccelerationEval(
        [pa], [pb.SummationDensity(dest='f', sources=['f'])],
        pb.CubicSpline(dim=2), backend=be)
    with pytest.raises(B200Error):
        ae.compute(0.0, 0.0)
    with pytest.raises(NotImplementedError):
        class Foo(pb.Equation):
            pass
        pb.B200AccelerationEval([pa], [Foo(dest='f', sources=['f'])],
                                pb.CubicSpline(dim=2), backend=be)
    # every property id through every entry point that names one
    f64 = set(range(0, 16)) | set(range(27, 32)) | set(range(70, 82)) | set(range(110, 126))
    f32 = set(range(16, 27)) | set(range(32, 38)) | set(range(82, 103))
    u32 = {64, 65, 66}
    accepts = dict(push_f64=f64 | f32, pull_f64=f64 | f32, push_u32=u32, pull_u32=u32,
                   device_ptr=f64 | f32 | u32, snapshot=f64 | f32 | u32)
    for entry, ids in accepts.items():
        rows, init = property_id_sweep(entry)
        assert [p for p, ok, _, _, _ in rows if ok] == sorted(ids), entry
        for p, ok, before, after, out in rows:
            # naming an elastic-dynamics property (70 .. 102) allocates the group: the ghost and
            # migration messages grow from 9 / 17 to 16 / 30 fields
            grows = entry not in ('push_u32', 'pull_u32')
            assert before == ((16, 30) if grows and p > 70 else (9, 17)), (entry, p)
            assert after == ((16, 30) if grows and p >= 70 else (9, 17)), (entry, p)
            if not ok:
                continue
            if entry == 'device_ptr':
                assert out, p
                continue
            if entry == 'push_f64':
                want = p + np.arange(5) / 3.0
            elif entry == 'push_u32':
                want = 1000 * p + np.arange(5)
            else:   # what the context was created with; zeros for what it was not given
                want = init.get(p, np.zeros(5))
            if p in f32:
                want = np.asarray(want, dtype=np.float32)
            assert np.array_equal(out, want), (entry, p, out, want)


SWEEP_IDS = list(range(-1, 127)) + [130, 255, 1 << 20]


def property_id_sweep(entry, skip=()):
    """What one entry point does with every property id in SWEEP_IDS (ascending), on a fresh
    context over one 5-particle array: rows (id, accepted, b200sph_halo_layout before and after,
    the values a push_f64 / pull_f64 or push_u32 / pull_u32 round trip, a pull or a one-segment
    snapshot returns, or whether device_ptr gave a pointer), and the values the context was
    created with, by id."""
    import ctypes as C
    import pysph_b200 as pb
    from pysph_b200._lib import B200Error, INT_PROP_IDS
    n = 5
    rs = np.random.RandomState(11)
    pa = pb.get_particle_array_wcsph(name='f', x=np.zeros(n))
    for k, a in pa.properties.items():
        a[:] = np.arange(n) + 7 if a.dtype.kind in 'iu' else rs.uniform(-2, 2, n)
    be = pb.B200Backend([pa])
    ids = dict(be.prop_ids[0], **INT_PROP_IDS)
    init = dict((ids[k], a.copy()) for k, a in pa.properties.items() if k in ids)
    call = be.ctx.call

    def layout():
        h, m = C.c_int(), C.c_int()
        call('b200sph_halo_layout', C.byref(h), C.byref(m))
        return h.value, m.value
    rows = []
    for p in SWEEP_IDS:
        if p in skip:
            continue
        before = layout()
        out = np.zeros(n, dtype=np.uint32 if entry.endswith('u32') else np.float64)
        try:
            if entry == 'push_f64':
                v = p + np.arange(n) / 3.0
                call('b200sph_push_f64', 0, p, v.ctypes.data, 0, n)
            elif entry == 'push_u32':
                v = (1000 * p + np.arange(n)).astype(np.uint32)
                call('b200sph_push_u32', 0, p, v.ctypes.data, 0, n)
            if entry == 'device_ptr':
                ptr = C.c_void_p()
                call('b200sph_device_ptr', 0, p, C.byref(ptr))
                out = ptr.value is not None
            elif entry == 'snapshot':
                call('b200sph_snapshot_take', 1, (C.c_int * 1)(0), (C.c_int * 1)(p),
                     (C.c_int64 * 1)(n))
                if p in INT_PROP_IDS.values():
                    out = out.astype(np.uint32)
                call('b200sph_snapshot_fetch', 0, out.ctypes.data, n)
                call('b200sph_snapshot_release')
            else:
                call('b200sph_pull_' + entry[-3:], 0, p, out.ctypes.data, 0, n)
            ok = True
        except B200Error:
            ok, out = False, None
        rows.append((p, ok, before, layout(), out))
    be.ctx.close()
    return rows, init


def test_determinism(gpu_device):
    """Two builds + evaluations of the same state give bit-identical results
    (the counting sort is made canonical inside each cell)."""
    from pysph_b200 import geometry as geo
    dx = 0.06
    res = []
    for _ in range(2):
        pas = geo.dam_break_3d_particles(dx=dx)
        rs = np.random.RandomState(3)
        for pa in pas[:1]:
            pa.u[:] = rs.normal(size=pa.u.size)
            pa.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, pa.u.size)
        s = make_solver(pas, scheme_params(geo.dam_break_3d_params(dx)),
                        'CubicSpline')
        s.initialise()
        s.step()
        s.pull()
        res.append(np.concatenate([pas[0].au, pas[0].arho, pas[0].x]))
    assert np.array_equal(res[0], res[1])


def test_size_independent_properties_100k(gpu_device):
    """At a size the oracle would take too long for in CI: lattice symmetry
    properties of config 2 at the example's default dx = 0.02 (~81 k fluid, 1/dx
    integer so that the lattice is mirror symmetric in y).
    * the initial state is mirror symmetric in y: au(y) = au(-y), av(y) = -av(-y)
    * interior fluid particles at rest: arho = 0, ax = u = 0
    * pair count is symmetric: #(fluid<-boundary) == #(boundary<-fluid)
    """
    import ctypes as C
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo, _lib
    dx = 0.02
    pas = geo.dam_break_3d_particles(dx=dx)
    params = geo.dam_break_3d_params(dx)
    s = make_solver(pas, scheme_params(params), 'CubicSpline')
    s.initialise()
    s.pull()
    f = pas[0]
    key = np.lexsort((np.round(f.z / dx), np.round(np.abs(f.y) / dx),
                      np.round(f.x / dx)))
    # pair up y-mirror images: particles with equal (x, |y|, z)
    xs, ys, zs = f.x[key], f.y[key], f.z[key]
    same = (np.abs(xs[1:] - xs[:-1]) < 1e-9) & (np.abs(zs[1:] - zs[:-1]) < 1e-9) & \
        (np.abs(ys[1:] + ys[:-1]) < 1e-9)
    i0, i1 = key[:-1][same], key[1:][same]
    assert len(i0) > 0.4 * f.x.size
    g = 9.81
    assert np.max(np.abs(f.au[i0] - f.au[i1])) <= 2e-4 * g
    assert np.max(np.abs(f.aw[i0] - f.aw[i1])) <= 2e-4 * g
    assert np.max(np.abs(f.av[i0] + f.av[i1])) <= 2e-4 * g
    assert np.max(np.abs(f.arho)) <= 1e-3     # fluid at rest: v_ij = 0 exactly
    assert np.max(np.abs(f.ax)) == 0.0
    # pair-count symmetry through two single-loop programs
    be = s.backend
    prog = _lib.PairProgram()
    cnt = C.c_int64()
    prog.eqmask[0][1] = _lib.EQ_CONTINUITY
    prog.real_only = 1
    be.ctx.call('b200sph_pair_pass', C.byref(prog), C.byref(cnt))
    n_fb = cnt.value
    prog = _lib.PairProgram()
    prog.eqmask[1][0] = _lib.EQ_CONTINUITY
    prog.real_only = 1
    be.ctx.call('b200sph_pair_pass', C.byref(prog), C.byref(cnt))
    assert n_fb == cnt.value and n_fb > 0


def _perturbed_dam_break(dx=0.05, vscale=0.5, seed=9):
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    rs = np.random.RandomState(seed)
    f = pas[0]
    for k in ('u', 'v', 'w'):
        f.properties[k][:] = rs.normal(scale=vscale, size=f.u.size)
    f.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, f.u.size)
    return pas, geo.dam_break_3d_params(dx)


def test_all_pair_kernels_agree(gpu_device, monkeypatch):
    """The two pair-kernel paths -- persistent neighbour lists (default) and the
    warp-per-destination kernel (fallback, also used for > 2^26 particles) --
    implement the same accept test and arithmetic: identical pair counts, results
    within fp32 summation-order noise, on a perturbed 3-D dam break."""
    out = {}
    for which in ('list', 'warp'):
        monkeypatch.setenv('B200SPH_PAIR_KERNEL', which)
        pas, params = _perturbed_dam_break()
        f = pas[0]
        s = make_solver(pas, scheme_params(params), 'CubicSpline')
        s.a_eval.count_pairs = True
        s.initialise()
        pairs = s.a_eval.last_pairs
        s.step()
        s.pull()
        out[which] = (pairs, dict((k, f.properties[k].copy())
                                  for k in ACC_FIELDS + ['x', 'u', 'rho']))
    for which in ('warp',):
        assert out['list'][0] == out[which][0]
        for k, v in out['list'][1].items():
            w = out[which][1][k]
            scale = max(np.max(np.abs(v)), 1e-30)
            assert np.max(np.abs(v - w)) <= 5e-6 * scale, (which, k)


def test_list_reuse_is_exact(gpu_device, monkeypatch):
    """Persistent lists with a skin give the same trajectory as rebuilding the
    neighbours at every evaluation (skin 0), and as the fp64 oracle, over enough
    fast steps that particles cross the skin several times."""
    res = {}
    for skin in ('0.1', '0.0'):
        monkeypatch.setenv('B200SPH_SKIN', skin)
        monkeypatch.setenv('B200SPH_PAIR_KERNEL', 'list')
        pas, params = _perturbed_dam_break(vscale=3.0)
        s = make_solver(pas, scheme_params(params), 'CubicSpline')
        for _ in range(40):
            s.step()
        s.pull()
        st = s.backend.stats()
        res[skin] = (pas, st, s.t)
    st = res['0.1'][1]
    assert st['light_updates'] > 20, st          # lists really were reused ...
    assert st['full_builds'] >= 3, st            # ... and rebuilt when the skin was used up
    # the integrator defers the drift check: each of those rebuilds followed a failed
    # check (evaluation repeated) or, when the extrapolated drift announced the failure, was
    # done one evaluation early
    assert st['deferred_failed'] + st['proactive_builds'] >= 2, st
    assert res['0.0'][1]['light_updates'] <= 2   # only updates with no motion at all
    pas_a, pas_b = res['0.1'][0], res['0.0'][0]
    assert abs(res['0.1'][2] - res['0.0'][2]) <= 1e-6 * res['0.0'][2]
    params = _perturbed_dam_break()[1]
    _compare_state(pas_a, pas_b, tol_pos=2e-6, tol_vel=2e-6, tol_rho=2e-7,
                   h0=params['h0'], c0=params['c0'], rho0=params['rho0'])
    # and against the oracle
    opas, _ = _perturbed_dam_break(vscale=3.0)
    o = orc.WCSPHOracleSolver(opas, params, 'CubicSpline', threads=4)
    for _ in range(40):
        o.step()
    _compare_state(pas_a, opas, tol_pos=2e-6, tol_vel=2e-6, tol_rho=2e-7,
                   h0=params['h0'], c0=params['c0'], rho0=params['rho0'])


def test_deferred_drift_check_protocol(gpu_device):
    """b200sph_nnps_update_deferred / b200sph_nnps_confirm (include/b200sph.h):
    a deferred update on stale lists evaluates garbage, confirm() says redo, the
    repeat equals a fresh evaluation; consuming an unconfirmed stale evaluation
    is an error, never a silent wrong answer."""
    import pysph_b200 as pb
    pas, params = _perturbed_dam_break()
    s = make_solver(pas, scheme_params(params), 'CubicSpline')
    s.initialise()                           # builds the lists
    be, nn, ae = s.backend, s.nnps, s.a_eval
    f = pas[0]
    # small motion: deferred update is confirmed
    f.x[:] += 1e-4 * params['h0']
    be.push(0, ['x'])
    nn.update(deferred=True)
    ae.compute(0.0, 0.0)
    assert nn.confirm() is False
    # a jump of one smoothing length: the lists are stale
    rs = np.random.RandomState(1)
    f.x[:] += params['h0'] * rs.uniform(-1, 1, f.x.size)
    be.push(0, ['x'])
    nn.update(deferred=True)
    ae.compute(0.0, 0.0)
    assert nn.confirm() is True
    assert nn.confirm() is False             # answered once
    nn.update()
    ae.compute(0.0, 0.0)
    be.pull_all(['au', 'arho', 'gid'])
    got = dict((k, f.properties[k][np.argsort(f.gid)].copy()) for k in ('au', 'arho'))
    # reference: a fresh context on the same state
    s.pull()
    q = copy_arrays(pas)
    s2 = make_solver(q, scheme_params(params), 'CubicSpline')
    s2.initialise()
    s2.pull()
    for k in ('au', 'arho'):
        ref = q[0].properties[k][np.argsort(q[0].gid)]
        assert rel_err(got[k], ref) <= 2e-6, k
    # unconfirmed stale update: stage / pull / dt_factors refuse
    f.x[:] += params['h0'] * rs.uniform(-1, 1, f.x.size)
    be.push(0, ['x'])
    nn.update(deferred=True)
    ae.compute(0.0, 0.0)
    with pytest.raises(RuntimeError, match='never confirmed'):
        be.pull(0, ['au'])
    assert be.stats()['deferred_failed'] == 2


def test_device_resident_dt_is_bitwise_the_host_path(gpu_device):
    """include/b200sph.h "device-resident time step": dt_propose / dt_commit /
    stage_dev perform the fp64 arithmetic of Integrator.compute_time_step and
    Solver._get_timestep (integrator.py:161-200, solver.py:647-688) on the
    device; with deterministic kernels the trajectory, t and dt are bitwise
    those of the host path, through the damped start-up and a tf-limited
    solve()."""
    out = {}
    for mode in (True, False):
        pas, params = _perturbed_dam_break(vscale=1.0)
        p = scheme_params(params)
        p['n_damp'] = 10
        s = make_solver(pas, p, 'CubicSpline', device_dt=mode)
        s.initialise()
        assert s.integrator.device_dt is mode
        dt0 = s.dt
        for _ in range(25):
            s.step()
        t25, dt25 = s.t, s.dt
        s.tf = t25 + 4.5 * dt25             # ends by time, not by count
        s.solve(1000)
        s.pull()
        out[mode] = (dt0, t25, dt25, s.count, s.t,
                     dict((k, pas[0].properties[k].copy()) for k in ('x', 'y', 'z', 'u', 'rho')))
    a, b = out[True], out[False]
    assert a[:5] == b[:5], (a[:5], b[:5])
    assert 27 <= a[3] <= 40
    for k, v in a[5].items():
        assert np.array_equal(v, b[5][k]), k


@pytest.mark.parametrize('idx', range(2))
def test_laminar_viscosity_vs_reference_bodies(gpu_device, idx):
    """WCSPHScheme(nu != 0): the WCSPH Group with LaminarViscosity (wc/viscosity.py:5-27,
    scheme.py:486-496) against the outputs of the reference's bodies (laminar_cases.json)."""
    import pysph_b200 as pb
    case = load_golden('laminar_cases.json')[idx]
    p = wcsph_params_from_case(case)
    pas = arrays_from_dict(case['inputs'])
    s = make_solver(pas, dict(scheme_params(p), nu=p['nu']), case['kernel'])
    names = [type(e).__name__ for e in s.a_eval.equation_groups[-1].equations]
    assert names[-2:] == ['LaminarViscosity', 'XSPHCorrection']      # inserted before XSPH
    s.a_eval.count_pairs = True
    s.a_eval.compute(0.0, 0.0)
    s.pull()
    opas = arrays_from_dict(case['inputs'])
    osol = orc.WCSPHOracleSolver(opas, p, case['kernel'])
    assert s.a_eval.last_pairs == osol.evaluate()
    visc_seen = False
    for pa, opa in zip(pas, opas):
        ref = case['outputs'][pa.name]
        nr = ref['_n_real']
        for f in ACC_FIELDS:
            want = np.array(ref[f])[:nr]
            got = pa.properties[f][:nr]
            if np.max(np.abs(want)) == 0.0:
                assert np.max(np.abs(got)) == 0.0, (pa.name, f)
                continue
            assert rel_err(got, want) <= TOL_EVAL, (pa.name, f, rel_err(got, want))
    # the viscous term is not lost in the tolerance: without it au differs by far more
    inv = load_golden('wcsph_cases.json')[0 if idx == 0 else 2]
    if idx == 0:
        d = np.array(case['outputs']['fluid']['au']) - np.array(inv['outputs']['fluid']['au'])
        assert np.max(np.abs(d)) > 1e-3 * np.max(np.abs(case['outputs']['fluid']['au']))


@pytest.mark.parametrize('idx', range(2))
def test_monaghan_av_vs_reference_bodies(gpu_device, idx):
    """The B200SPH_EQ_MONAGHAN_AV branch of pair_body: a Group with ContinuityEquation,
    stand-alone MonaghanArtificialViscosity (basic_equations.py:195-257) and
    XSPHCorrection, against the values the reference's own bodies produced
    (tests/golden/monaghan_av_cases.json, oracle/gen_golden.py)."""
    import pysph_b200 as pb
    from test_oracle_golden import run_oracle_monaghan_case
    case = load_golden('monaghan_av_cases.json')[idx]
    p = case['params']
    names = p['names']
    pas = arrays_from_dict(case['inputs'], order=tuple(names))
    kernel = getattr(pb, case['kernel'])(dim=case['dim'])
    groups = [
        pb.Group(equations=[pb.TaitEOS(dest=a, sources=None, rho0=p['rho0'], c0=p['c0'],
                                       gamma=p['gamma']) for a in names], real=False),
        pb.Group(equations=[
            pb.ContinuityEquation(dest='fluid', sources=names),
            pb.MonaghanArtificialViscosity(dest='fluid', sources=names, alpha=p['alpha'],
                                           beta=p['beta']),
            pb.XSPHCorrection(dest='fluid', sources=['fluid'], eps=p['eps_xsph'])],
            real=True)]
    ae = pb.B200AccelerationEval(pas, groups, kernel)
    nn = pb.B200NNPS(case['dim'], pas, backend=ae.backend, kernel=kernel)
    ae.set_nnps(nn)
    ae.count_pairs = True
    ae.compute(0.0, 0.0)
    ae.backend.pull_all()
    _, pairs = run_oracle_monaghan_case(case)
    assert ae.last_pairs == pairs
    ref = case['outputs']['fluid']
    nr = ref['_n_real']
    for f in ('arho', 'au', 'av', 'aw', 'ax', 'ay', 'az'):
        want = np.array(ref[f])[:nr]
        assert rel_err(pas[0].properties[f][:nr], want) <= TOL_EVAL, f
    assert np.max(np.abs(ref['au'])) > 1.0


@pytest.mark.parametrize('device_dt', [True, False])
def test_fused_stage_kernel_is_bitwise_the_separate_kernels(gpu_device, monkeypatch, device_dt, dx=0.05):
    """include/b200sph.h "Fast path" of b200sph_stage / b200sph_stage_dev: k_stage_pack (stage
    + packed records of the next evaluation with the last evaluation's EOS calls applied
    speculatively + drift of the build + dt factors) against k_stage, k_pack_pos_light,
    k_pack_state and k_reduce_dt run one after the other (B200SPH_FUSE=0): every property
    the host can pull -- including p / cs / rho of the HG-corrected solids and the stage
    copies x0 .. rho0 -- t, dt and the rebuild count must be bitwise equal through list
    rebuilds (3 m/s random velocities use up the skin in a few steps)."""
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        pas, params = _perturbed_dam_break(dx=dx, vscale=3.0)
        p = scheme_params(params)
        p['n_damp'] = 6
        s = make_solver(pas, p, 'CubicSpline', device_dt=device_dt)
        for _ in range(22):
            s.step()
        st = s.backend.stats()
        s.pull()
        out[fuse] = (s.t, s.dt, st['full_builds'],
                     [dict((k, v.copy()) for k, v in pa.properties.items()) for pa in pas])
        if fuse == '1':
            assert st['full_builds'] >= 2          # the lists were rebuilt on the way
            assert st['fused_stages'] >= 30        # ... and the fused kernel served the stages
        else:
            assert st['fused_stages'] == 0
    a, b = out['1'], out['0']
    assert a[:3] == b[:3], (a[:3], b[:3])
    for pa, pb_ in zip(a[3], b[3]):
        for k, v in pa.items():
            assert np.array_equal(v, pb_[k]), k


def test_zorder_rows_give_the_same_neighbours_and_fields(gpu_device, monkeypatch):
    """B200SPH_ZORDER=1 orders the cell rows along the Z-curve of (cy, cz) (north_star's
    "Z-curve cell list"; z_order_nnps.pyx:252-355 sorts by the 3-D Morton key): only the
    order in which neighbours are visited changes -- identical pair counts, neighbour sets
    and (to fp32 summation order) fields, through list rebuilds.  In either order one
    evaluation of a coarser perturbed dam break matches the oracle: pair count, every
    acceleration-like field, p and cs."""
    import pysph_b200 as pb
    opas, oparams = _perturbed_dam_break(dx=0.09, seed=5)
    o = orc.WCSPHOracleSolver(opas, oparams, 'CubicSpline')
    want_pairs = o.evaluate()
    out = {}
    for z in ('0', '1'):
        monkeypatch.setenv('B200SPH_ZORDER', z)
        pas, params = _perturbed_dam_break(dx=0.09, seed=5)
        s = make_solver(pas, scheme_params(params), 'CubicSpline')
        s.a_eval.count_pairs = True
        s.a_eval.compute(0.0, 0.0)
        s.pull()
        assert s.a_eval.last_pairs == want_pairs, z
        for pa, oa in zip(pas, opas):
            for k in ACC_FIELDS + ['p', 'cs']:
                err = rel_err(pa.properties[k], oa.properties[k])
                assert err <= TOL_EVAL, (z, pa.name, k, err)
        pas, params = _perturbed_dam_break(vscale=3.0)
        s = make_solver(pas, scheme_params(params), 'CubicSpline')
        s.a_eval.count_pairs = True
        s.initialise()
        pairs = s.a_eval.last_pairs
        nn = s.nnps
        nb = [np.sort(nn.get_nearest_particles(0, d, i)) for d in range(3)
              for i in (0, pas[d].get_number_of_particles() // 2, pas[d].get_number_of_particles() - 1)]
        s.a_eval.count_pairs = False
        for _ in range(22):
            s.step()
        st = s.backend.stats()
        s.pull()
        out[z] = (pairs, nb, st['full_builds'],
                  dict((k, pas[0].properties[k].copy()) for k in ACC_FIELDS + ['x', 'u', 'rho']))
    assert out['0'][0] == out['1'][0] and out['0'][2] == out['1'][2] >= 2
    for a, b in zip(out['0'][1], out['1'][1]):
        assert np.array_equal(a, b)
    for k, v in out['0'][3].items():
        w = out['1'][3][k]
        assert np.max(np.abs(v - w)) <= 5e-6 * max(np.max(np.abs(v)), 1e-30), k
