"""A destroyed context gives back every device and pinned buffer it allocated, the lazily grown
ones included, on the emulated library (tests/test_library_on_cpu.py): the emulation's allocator
counts its live blocks."""
import ctypes as C

import numpy as np

from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _lattice(nx, dx):
    g = (np.arange(nx) + 0.5) * dx
    x, y, z = np.meshgrid(g, g, g, indexing='ij')
    return x.ravel(), y.ravel(), z.ravel()


def test_destroy_frees_every_buffer(emulated_library):
    from pysph_b200 import _lib
    lib = _lib.load()
    live = lib.emu_live_blocks
    live.restype = C.c_longlong
    ids = _lib.PROP_IDS
    before = live()

    ctx = _lib.Context(0)
    nx, dx = 8, 0.1
    x, y, z = _lattice(nx, dx)
    n = x.size
    ctx.call('b200sph_add_array', b'fluid', n, n, n)
    state = dict(x=x, y=y, z=z, u=np.zeros(n), v=np.zeros(n), w=np.zeros(n), rho=np.full(n, 1000.0),
                 h=np.full(n, 1.3 * dx), m=np.full(n, 1000.0 * dx ** 3))
    for k, a in state.items():
        ctx.call('b200sph_push_f64', 0, ids[k], _ptr(a), 0, n)
    # an fp32 property goes through the staging buffer both ways
    p = np.linspace(0.0, 1.0, n)
    ctx.call('b200sph_push_f64', 0, ids['p'], _ptr(p), 0, n)
    ctx.call('b200sph_pull_f64', 0, ids['p'], _ptr(p), 0, n)
    ctx.call('b200sph_set_kernel', 0, 3)

    # an NNPS update and a pair pass over the lists (scan scratch, cells, lists)
    prog = _lib.PairProgram()
    prog.eqmask[0][0] = _lib.EQ_SUMMATION_DENSITY | _lib.EQ_CONTINUITY | _lib.EQ_MOMENTUM
    prog.c0 = 10.0
    pairs = _lib._i64()

    def evaluate():
        ctx.call('b200sph_nnps_update')
        ctx.call('b200sph_pair_pass', C.byref(prog), C.byref(pairs))
        assert pairs.value > 0
    evaluate()

    # the device-resident time-control block and its pinned snapshot slots
    ctx.call('b200sph_time_control', None, None)

    # an output snapshot: take, fetch, release
    segs = 3
    arr = (C.c_int * segs)(0, 0, -1)
    prop = (C.c_int * segs)(ids['x'], ids['p'], 0)
    count = (_lib._i64 * segs)(n, n, 2)
    ctx.call('b200sph_snapshot_take', segs, arr, prop, count)
    got = np.zeros(n)
    ctx.call('b200sph_snapshot_fetch', 0, _ptr(got), n)
    assert np.array_equal(got, x)
    ctx.call('b200sph_snapshot_release')

    # get_neighbors (its scratch is a temporary)
    nbrs = np.zeros(256, dtype=np.uint32)
    assert ctx.call('b200sph_get_neighbors', 0, 0, 0, _ptr(nbrs), nbrs.size) > 0

    # the density filter (its records), with rhotmp a user property
    rhotmp = _lib.USER_PROP0
    ctx.call('b200sph_user_property', rhotmp)
    ctx.call('b200sph_density_filter', 1, _lib.DFILTER_SHEPARD, 0, rhotmp, 0)

    # probe sets and the interpolator's scratch; the second set is still alive at the destroy
    q = np.linspace(0.2, 0.6, 7)
    props = (C.c_int * _lib.MAX_ARRAYS)(*([ids['rho']] + [-1] * (_lib.MAX_ARRAYS - 1)))
    out = np.zeros(4 * q.size)
    for method in ('shepard', 'order1'):
        pid = ctx.call('b200sph_probe_create', q.size, _ptr(q), _ptr(q), _ptr(q), 1.3 * dx)
        ctx.call('b200sph_interpolate', pid, _lib.INTERP_METHODS[method], 0, 3, props, 1, _ptr(out))
        if method == 'shepard':
            assert np.all(out[:q.size] > 0.0)
            ctx.call('b200sph_probe_release', pid)

    # halo selections for both neighbours, ghosts appended (the pool grows), and a list
    # rebuild with ghosts, which splits the list consumer's chunks
    bufs, counts = [], []
    for slot, (lo, hi) in enumerate(((0.0, 2 * dx), (0.6, 0.8))):
        buf = np.zeros(9 * n)
        cnt = _lib._i64()
        ctx.call('b200sph_halo_pack', 0, slot, lo, hi, _ptr(buf), n, C.byref(cnt))
        assert cnt.value > 0
        bufs.append(buf)
        counts.append(cnt.value)
    ghosts = bufs[0][:9 * counts[0]].copy()
    ghosts[:counts[0]] += nx * dx          # beyond the right end of the block
    ctx.call('b200sph_halo_append', 0, _ptr(ghosts), counts[0], counts[0], _lib.HALO_FIELDS, 0)
    evaluate()
    stats = _lib.Stats()
    ctx.call('b200sph_get_stats', C.byref(stats))
    assert stats.chunks_boundary > 0

    # mirror images (they replace the ghosts)
    lo = (C.c_double * 3)(-0.05, -0.05, -0.05)
    hi = (C.c_double * 3)(nx * dx + 0.05, nx * dx + 0.05, nx * dx + 0.05)
    ctx.call('b200sph_set_domain', lo, hi, (C.c_int * 3)(0, 0, 0))
    ctx.call('b200sph_set_mirror', (C.c_int * 3)(1, 0, 0), 2.0)
    evaluate()
    n_all, n_real = _lib._i64(), _lib._i64()
    ctx.call('b200sph_get_array_size', 0, C.byref(n_all), C.byref(n_real))
    assert n_real.value == n and n_all.value > n

    # an elastic-dynamics property: the elastic group with its stress records
    s00 = np.zeros(n)
    ctx.call('b200sph_push_f64', 0, _lib.ELASTIC_PROP_IDS['s00'], _ptr(s00), 0, n)

    assert live() > before
    ctx.close()
    assert live() == before
