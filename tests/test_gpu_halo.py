"""Single-GPU tests of the halo / migration entry points of the C-ABI (the device
side of the slab decomposition, include/b200sph.h "halo exchange helpers"),
checked against numpy on the same data."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F9 = ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'h', 'm']
F16 = F9 + ['x0', 'y0', 'z0', 'u0', 'v0', 'w0', 'rho0']


def _array(name, n, seed):
    import pysph_b200 as pb
    rs = np.random.RandomState(seed)
    props = dict((k, rs.uniform(0.1, 1.0, n)) for k in F16)
    props['x'] = rs.uniform(0.0, 3.0, n)
    pa = pb.get_particle_array_wcsph(name=name, **props)
    pa.gid[:] = np.arange(n) + 1000 * seed
    return pa


def test_halo_pack_append_overwrite_migrate(gpu_device):
    import pysph_b200 as pb
    from pysph_b200.parallel import DeviceHaloOps, HALO_FIELDS, MIGRATE_FIELDS
    a, b = _array('fluid', 500, 1), _array('wall', 200, 2)
    ref = [dict((k, v.copy()) for k, v in p.properties.items()) for p in (a, b)]
    be = pb.B200Backend([a, b], extra_capacity=2000)
    ops = DeviceHaloOps(be, 0)

    # -- halo_pack: lo <= x < hi of the real particles, field-major and tight
    lo, hi = 1.0, 1.6
    buf = ops.new_buffer(9 * 700)
    n = ops.pack(0, 1, lo, hi, buf, 0)
    sel = np.where((ref[0]['x'] >= lo) & (ref[0]['x'] < hi))[0]
    assert n == sel.size and n > 20
    got = buf[:9 * n].cpu().numpy().reshape(9, n)
    for f, k in enumerate(F9):
        assert np.array_equal(got[f], ref[0][k][sel]), k   # stable order, exact fp64

    # -- append as ghosts: n grows, n_real does not; ghosts carry the 9 fields, tag 1
    ops.append(1, buf, 0, n, HALO_FIELDS, False)
    assert be.sizes(1) == (200 + n, 200)
    be.pull(1)
    for f, k in enumerate(F9):
        assert np.array_equal(b.properties[k][200:], ref[0][k][sel]), k
    assert np.all(b.tag[200:] == 1) and np.all(b.tag[:200] == 0)
    assert np.all(b.x0[200:] == 0.0) and np.all(b.gid[200:] == 2 ** 32 - 1)
    assert np.array_equal(b.x[:200], ref[1]['x'])

    # -- pack_selected returns the CURRENT values of the remembered particles
    a.rho[:] = ref[0]['rho'] + 5.0
    be.push(0, ['rho'])
    buf2 = ops.new_buffer(9 * 700)
    assert ops.pack_selected(0, 1, buf2, 0) == n
    got2 = buf2[:9 * n].cpu().numpy().reshape(9, n)
    assert np.array_equal(got2[6], ref[0]['rho'][sel] + 5.0)
    assert np.array_equal(got2[0], ref[0]['x'][sel])

    # -- overwrite the ghosts in place
    ops.overwrite(1, 0, buf2, 0, n)
    be.pull(1, ['rho', 'x'])
    assert np.array_equal(b.rho[200:], ref[0]['rho'][sel] + 5.0)
    assert be.sizes(1) == (200 + n, 200)
    with pytest.raises(RuntimeError):
        ops.overwrite(1, 1, buf2, 0, n)          # past the last ghost

    # -- drop_ghosts
    ops.drop_ghosts(1)
    assert be.sizes(1) == (200, 200)

    # -- migrate_out: particles outside [lo, hi) leave, the rest is compacted in order
    mlo, mhi = 0.5, 2.5
    mbuf = ops.new_buffer(MIGRATE_FIELDS * 500)
    n_lo, n_hi = ops.migrate_out(0, mlo, mhi, mbuf, 0)
    x = ref[0]['x']
    s_lo, s_hi = np.where(x < mlo)[0], np.where(x >= mhi)[0]
    keep = np.where((x >= mlo) & (x < mhi))[0]
    assert (n_lo, n_hi) == (s_lo.size, s_hi.size) and n_lo > 0 and n_hi > 0
    blk_lo = mbuf[:17 * n_lo].cpu().numpy().reshape(17, n_lo)
    blk_hi = mbuf[17 * n_lo:17 * (n_lo + n_hi)].cpu().numpy().reshape(17, n_hi)
    cur = dict(ref[0])
    cur['rho'] = ref[0]['rho'] + 5.0
    for f, k in enumerate(F16):
        assert np.array_equal(blk_lo[f], cur[k][s_lo]), k
        assert np.array_equal(blk_hi[f], cur[k][s_hi]), k
    assert np.array_equal(blk_lo[16], ref[0]['gid'][s_lo].astype(float))
    assert be.sizes(0) == (keep.size, keep.size)
    be.pull(0)
    for k in F16:
        assert np.array_equal(a.properties[k], cur[k][keep]), k
    assert np.array_equal(a.gid, ref[0]['gid'][keep])

    # -- the migrants arrive somewhere as REAL particles with all 16 fields + gid
    ops.append(1, mbuf, 0, n_lo, MIGRATE_FIELDS, True)
    assert be.sizes(1) == (200 + n_lo, 200 + n_lo)
    be.pull(1)
    for k in F16:
        assert np.array_equal(b.properties[k][200:], cur[k][s_lo]), k
    assert np.array_equal(b.gid[200:], ref[0]['gid'][s_lo])
    assert np.all(b.tag[200:] == 0)


def test_evaluation_with_ghosts_equals_one_array(gpu_device):
    """Group(real=True) semantics with ghosts (acceleration_eval_cython_helper.py
    :271-286): split one fluid block into a 'real' part and ghosts imported with
    halo_append -- the real particles get exactly the accelerations of the
    unsplit evaluation (same neighbours, same order up to the sort)."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from pysph_b200.parallel import DeviceHaloOps, HALO_FIELDS
    dx = 0.06
    params = geo.dam_break_3d_params(dx)
    pas = geo.dam_break_3d_particles(dx=dx)
    rs = np.random.RandomState(4)
    f = pas[0]
    f.u[:] = rs.normal(size=f.u.size)
    f.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, f.u.size)
    whole = pb.make_wcsph_solver(pas, dict(params), pb.CubicSpline(dim=3))
    whole.initialise()
    whole.pull()
    ref = dict((k, f.properties[k].copy()) for k in ('au', 'av', 'aw', 'arho', 'ax', 'gid'))

    # same state, but the fluid with x >= cut lives in a donor array and is imported
    cut = 0.6
    pas2 = geo.dam_break_3d_particles(dx=dx)
    f2 = pas2[0]
    f2.u[:] = f.u
    f2.rho[:] = f.rho
    left = np.where(f2.x < cut)[0]
    right = np.where(f2.x >= cut)[0]
    fl = f2.extract(left, name='fluid')
    donor = f2.extract(right, name='donor')
    be = pb.B200Backend([fl, pas2[1], pas2[2], donor], extra_capacity=right.size + 64)
    ops = DeviceHaloOps(be, 0)
    buf = ops.new_buffer(9 * right.size)
    n = ops.pack(3, -1, -1e9, 1e9, buf, 0)
    assert n == right.size
    ops.append(0, buf, 0, n, HALO_FIELDS, False)
    be.ctx.call('b200sph_resize_array', 3, 0, 0)      # the donor array is emptied
    p = dict(params)
    for k in ('integrator', 'dt0', 'n_damp', 'cfl'):
        p.pop(k)
    scheme = pb.WCSPHScheme(**p)
    ae = pb.B200AccelerationEval([fl, pas2[1], pas2[2], donor], scheme.get_equations(),
                                 pb.CubicSpline(dim=3), backend=be)
    nn = pb.B200NNPS(3, [fl, pas2[1], pas2[2], donor], backend=be,
                     kernel=pb.CubicSpline(dim=3))
    ae.set_nnps(nn)
    ae.compute(0.0, 0.0)
    be.pull(0)
    nr = left.size
    assert be.sizes(0) == (left.size + right.size, nr)
    order = np.argsort(ref['gid'])
    pos = order[np.searchsorted(ref['gid'][order], fl.gid[:nr])]
    for k in ('au', 'av', 'aw', 'arho', 'ax'):
        scale = max(np.max(np.abs(ref[k])), 1e-30)
        assert np.max(np.abs(fl.properties[k][:nr] - ref[k][pos])) <= 5e-6 * scale, k
    # ghosts are sources only: their accelerations were never written
    assert np.all(fl.au[nr:] == 0.0)
