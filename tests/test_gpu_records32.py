"""The 32-byte pair records of the WCSPH pass (k_pair_list_r32) against the 48-byte ones
(B200SPH_RECORDS=48), and the conditions under which the library picks them.

The 32-byte records hold (x, y, z, rho / rho0 - 1, u, v, w, type): h and m must be uniform,
every array must carry the same Tait EOS (gamma = 7) and there must be no ghosts.  The
accept test runs on the same floats in both layouts, so pair counts are equal; p / rho^2 and
cs are recomputed per pair in fp32, so fields agree to fp32 rounding.
"""
import numpy as np
import pytest

from helpers import ACC_FIELDS

pytestmark = pytest.mark.gpu


def _state(dx, vscale=3.0, seed=9):
    """A dam break with random velocities and densities; the walls start below rho0 so that
    TaitEOSHGCorrection clamps them."""
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    rs = np.random.RandomState(seed)
    f = pas[0]
    for k in ('u', 'v', 'w'):
        f.properties[k][:] = rs.normal(scale=vscale, size=f.u.size)
    f.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, f.u.size)
    for pa in pas[1:]:
        pa.rho[:] *= 1 - 0.005 * rs.uniform(0, 1, pa.rho.size)
    return pas, geo.dam_break_3d_params(dx)


def _solver(pas, params, **kw):
    import pysph_b200 as pb
    keep = ('fluids', 'solids', 'dim', 'rho0', 'c0', 'h0', 'hdx', 'gamma', 'gx', 'gy', 'gz',
            'alpha', 'beta', 'tensile_correction', 'hg_correction', 'update_h',
            'summation_density', 'dt0', 'n_damp', 'cfl', 'integrator')
    p = dict((k, v) for k, v in params.items() if k in keep)
    return pb.make_wcsph_solver(pas, p, pb.CubicSpline(dim=3), **kw)


def _set_records(monkeypatch, which):
    if which == '48':
        monkeypatch.setenv('B200SPH_RECORDS', '48')
    else:
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)


def _run(monkeypatch, which, dx, steps, edit=None):
    _set_records(monkeypatch, which)
    pas, params = _state(dx)
    if edit:
        edit(pas)
    s = _solver(pas, params)
    s.a_eval.count_pairs = True
    s.initialise()
    pairs = s.a_eval.last_pairs
    s.a_eval.count_pairs = False
    s.pull()
    first = [dict((k, pa.properties[k].copy()) for k in ACC_FIELDS) for pa in pas]
    for _ in range(steps):
        s.step()
    s.pull()
    return dict(pairs=pairs, first=first, pas=pas, params=params, stats=s.backend.stats())


def test_records32_match_records48(gpu_device, monkeypatch, dx=0.05, steps=40):
    """Same pairs; accelerations of one evaluation within 5e-6 max|field|; the state after
    `steps` EPEC steps (list rebuilds on the way) within 2e-6 h0 / 2e-6 c0 / 2e-7 rho0."""
    r32 = _run(monkeypatch, '32', dx, steps)
    r48 = _run(monkeypatch, '48', dx, steps)
    assert r32['stats']['pair_launches_r32'] == r32['stats']['pair_launches'] > 0
    assert r48['stats']['pair_launches_r32'] == 0
    assert r32['stats']['full_builds'] >= 2, r32['stats']
    assert r32['pairs'] == r48['pairs'] > 0
    for a, b in zip(r32['first'], r48['first']):
        for k in ACC_FIELDS:
            scale = max(np.max(np.abs(b[k])), 1e-30)
            assert np.max(np.abs(a[k] - b[k])) <= 5e-6 * scale, k
    p = r48['params']
    for pa, pb_ in zip(r32['pas'], r48['pas']):
        for k in ('x', 'y', 'z'):
            assert np.max(np.abs(pa.properties[k] - pb_.properties[k])) <= 2e-6 * p['h0'], (pa.name, k)
        for k in ('u', 'v', 'w'):
            assert np.max(np.abs(pa.properties[k] - pb_.properties[k])) <= 2e-6 * p['c0'], (pa.name, k)
        assert np.max(np.abs(pa.rho - pb_.rho)) <= 2e-7 * p['rho0'], pa.name


def test_records32_fused_stage_is_bitwise_the_separate_kernels(gpu_device, monkeypatch, dx=0.05, steps=22):
    """k_stage_pack writing the 32-byte records and k_stage + k_pack_pos_light + k_pack_rec32
    (B200SPH_FUSE=0) give bitwise the same run, through list rebuilds."""
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        r = _run(monkeypatch, '32', dx, steps)
        st = r['stats']
        assert st['pair_launches_r32'] == st['pair_launches'] > 0
        assert (st['fused_stages'] > 0) == (fuse == '1')
        out[fuse] = r
    assert out['1']['pairs'] == out['0']['pairs']
    for pa, pb_ in zip(out['1']['pas'], out['0']['pas']):
        for k, v in pa.properties.items():
            assert np.array_equal(v, pb_.properties[k]), (pa.name, k)


def _perturb_h(pas):
    pas[0].h[3] *= 1.0001


def _perturb_m(pas):
    pas[1].m[5] *= 1.01


@pytest.mark.parametrize('edit', [_perturb_h, _perturb_m], ids=['h', 'm'])
def test_nonuniform_h_or_m_keeps_48_byte_records(gpu_device, monkeypatch, edit, dx=0.08, steps=4):
    """One particle with another h or m: the 48-byte records serve every pass, and the run
    is bitwise the one with B200SPH_RECORDS=48."""
    a = _run(monkeypatch, '32', dx, steps, edit)
    b = _run(monkeypatch, '48', dx, steps, edit)
    assert a['stats']['pair_launches_r32'] == 0 and a['stats']['pair_launches'] > 0
    for pa, pb_ in zip(a['pas'], b['pas']):
        for k, v in pa.properties.items():
            assert np.array_equal(v, pb_.properties[k]), (pa.name, k)


def test_pushed_mass_is_noticed(gpu_device, monkeypatch, dx=0.08):
    """A push of m that breaks uniformity switches the next evaluation back to 48-byte
    records; one that restores it switches to the 32-byte ones again."""
    _set_records(monkeypatch, '32')
    pas, params = _state(dx)
    s = _solver(pas, params)
    s.initialise()
    be = s.backend
    n0 = be.stats()['pair_launches_r32']
    assert n0 > 0
    m_old = pas[0].m[0]
    pas[0].m[0] = 2.0 * m_old
    be.push_real_array(0, ['m'])
    s.step()
    st = be.stats()
    assert st['pair_launches_r32'] == n0
    pas[0].m[0] = m_old
    be.push_real_array(0, ['m'])
    s.step()
    assert be.stats()['pair_launches_r32'] > n0


def test_ranged_group_takes_48_byte_records(gpu_device, monkeypatch, dx=0.08):
    """Group(start_idx, stop_idx) runs the RANGED k_pair_list on the 48-byte records, and the
    destinations outside the range are left alone."""
    from pysph_b200 import _lib
    import ctypes as C
    _set_records(monkeypatch, '32')
    pas, params = _state(dx)
    s = _solver(pas, params)
    s.initialise()
    be = s.backend
    n0 = be.stats()['pair_launches_r32']
    assert n0 > 0
    s.pull()
    au_before = pas[0].au.copy()
    prog = _lib.PairProgram()      # the fluid's WCSPH equations over the fluid only
    prog.eqmask[0][0] = _lib.EQ_CONTINUITY | _lib.EQ_MOMENTUM | _lib.EQ_XSPH
    prog.c0, prog.alpha, prog.beta = params['c0'], params['alpha'], params['beta']
    for a in range(len(pas)):
        be.ctx.call('b200sph_eos', a, int(a > 0), params['rho0'], params['c0'], 7.0, 0.0, 0)
    be.ctx.call('b200sph_set_dest_range', 0, 2, 5)
    be.ctx.call('b200sph_pair_pass', C.byref(prog), None)
    assert be.stats()['pair_launches_r32'] == n0
    s.pull()
    assert np.array_equal(pas[0].au[:2], au_before[:2])
    assert np.array_equal(pas[0].au[5:], au_before[5:])
