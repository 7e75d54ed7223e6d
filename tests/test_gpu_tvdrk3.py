"""TVDRK3Integrator + WCSPHTVDRK3Step (integrator.py:426-460, integrator_step.py:96-168) on
the device: the stepper against the reference's own body (tvdrk3_stepper.json), the fused
stage kernel (k_stage_pack_rk3) against the separate kernels bitwise, whole runs against the
fp64 oracle, the time control with three evaluations per step, and the refusals.

The check_* functions take the sizes as arguments: tests/test_tvdrk3_on_cpu.py runs the same
checks, smaller, on the library emulation.
"""
import os

import numpy as np
import pytest

from helpers import copy_arrays, load_golden
from tvdrk3_oracle import TVDRK3OracleSolver, stage_rk3

pytestmark = pytest.mark.gpu

STATE = ['x', 'y', 'z', 'u', 'v', 'w', 'rho']
STAGES = ((0, 'initialize'), (1, 'stage1'), (2, 'stage2'), (3, 'stage3'))


# ---- helpers ---------------------------------------------------------------------------------
def _dam_break(dx, vscale=0.0, seed=9):
    """The 3-D dam break; vscale > 0 adds random velocities that use up the list skin."""
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    if vscale:
        rs = np.random.RandomState(seed)
        f = pas[0]
        for k in ('u', 'v', 'w'):
            f.properties[k][:] = rs.normal(scale=vscale, size=f.u.size)
        f.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, f.u.size)
    return pas, dict(geo.dam_break_3d_params(dx), integrator='TVDRK3')


def _solver(pas, params, kernel='CubicSpline', **kw):
    import pysph_b200 as pb
    keep = ('fluids', 'solids', 'dim', 'rho0', 'c0', 'h0', 'hdx', 'gamma', 'gx', 'gy', 'gz',
            'alpha', 'beta', 'tensile_correction', 'hg_correction', 'update_h',
            'summation_density', 'dt0', 'n_damp', 'cfl', 'integrator')
    p = dict((k, v) for k, v in params.items() if k in keep)
    return pb.make_wcsph_solver(pas, p, getattr(pb, kernel)(dim=params['dim']), **kw)


def _compare_state(pas, opas, params, pos=2e-6, vel=2e-6, rho=2e-7):
    h0, c0, rho0 = params['h0'], params['c0'], params['rho0']
    for pa, oa in zip(pas, opas):
        n = oa.num_real_particles
        for k, tol in (('x', pos * h0), ('y', pos * h0), ('z', pos * h0), ('u', vel * c0),
                       ('v', vel * c0), ('w', vel * c0), ('rho', rho * rho0)):
            err = np.max(np.abs(pa.properties[k][:n] - oa.properties[k][:n]))
            assert err <= tol, (pa.name, k, err, tol)


def _run(pas, params, steps, kernel='CubicSpline', **kw):
    s = _solver(pas, params, kernel, **kw)
    for _ in range(steps):
        s.step()
    st = s.backend.stats()
    s.pull()
    return s, st


# ---- 1. the stepper against the reference's body ----------------------------------------------
def check_stepper_golden(tol=1e-14):
    """Every stage, on every array at once (arr = -1) and array by array, with dt from the host
    and from the time-control block, against WCSPHTVDRK3Step's own body; and the oracle's
    restatement of the stepper (tests/tvdrk3_oracle.py) the same way."""
    import pysph_b200 as pb
    g = load_golden('tvdrk3_stepper.json')
    n = len(g['inputs']['x'])
    cut = n // 2

    def arrays():
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        return [pb.get_particle_array_wcsph(name='a', **dict((k, v[:cut]) for k, v in props.items())),
                pb.get_particle_array_wcsph(name='b', **dict((k, v[cut:]) for k, v in props.items()))]

    def compare(pas, key, who):
        for k, want in g['outputs'][key].items():
            want = np.array(want)
            got = np.concatenate([pa.properties[k] for pa in pas])
            scale = max(np.max(np.abs(want)), 1e-300)
            assert np.max(np.abs(got - want)) <= tol * scale, (who, key, k)

    for which, key in STAGES:
        for per_array in (False, True):
            for devdt in (False, True):
                pas = arrays()
                be = pb.B200Backend(pas)
                if devdt:
                    be.ctx.call('b200sph_time_set', 0.0, g['dt'])
                for arr in ((0, 1) if per_array else (-1,)):
                    if devdt:
                        be.ctx.call('b200sph_stage_rk3_dev', arr, which)
                    else:
                        be.ctx.call('b200sph_stage_rk3', arr, which, g['dt'])
                be.pull_all()
                compare(pas, key, ('device', per_array, devdt))
        pas = arrays()
        for pa in pas:
            stage_rk3(pa, which, g['dt'])
        compare(pas, key, 'oracle')
    # stage1 of TVD-RK3 is a whole-dt step, not WCSPHStep's half step
    assert g['outputs']['stage1']['x'][0] == pytest.approx(
        g['inputs']['x0'][0] + g['dt'] * g['inputs']['ax'][0], rel=1e-15)


# ---- 2. fused == unfused, bitwise -----------------------------------------------------------
def check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx, steps=22, min_fused=30):
    """k_stage_pack_rk3 (stage + records of the next evaluation + drift + dt factors after
    stage3) against k_stage_rk3 + the separate packing kernels (B200SPH_FUSE=0): every pullable
    property, t, dt and the rebuild count bitwise, through list rebuilds."""
    if records == '48':
        monkeypatch.setenv('B200SPH_RECORDS', '48')
    else:
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        pas, params = _dam_break(dx, vscale=3.0)
        params['n_damp'] = 6
        s, st = _run(pas, params, steps, device_dt=device_dt)
        out[fuse] = (s.t, s.dt, st['full_builds'],
                     [dict((k, v.copy()) for k, v in pa.properties.items()) for pa in pas])
        if fuse == '1':
            assert st['full_builds'] >= 2, st             # the lists were rebuilt on the way
            assert st['fused_stages'] >= min_fused, st    # ... and the fused kernel served
            if records == '48':
                assert st['pair_launches_r32'] == 0, st
            else:
                assert st['pair_launches_r32'] == st['pair_launches'] > 0, st
        else:
            assert st['fused_stages'] == 0
    a, b = out['1'], out['0']
    assert a[:3] == b[:3], (a[:3], b[:3])
    for pa, pb_ in zip(a[3], b[3]):
        for k, v in pa.items():
            assert np.array_equal(v, pb_[k]), k


# ---- 3. whole runs against the oracle -------------------------------------------------------
def check_dam_break_3d_vs_oracle(dx, steps, vscale=0.0, threads=4):
    """Adaptive TVD-RK3 steps of the 3-D dam break (vscale > 0: random velocities force list
    rebuilds) against the oracle: same pairs, same dt sequence to 1e-6, the state within the
    EPEC bars."""
    pas, params = _dam_break(dx, vscale)
    opas = copy_arrays(pas)
    s = _solver(pas, params)
    o = TVDRK3OracleSolver(opas, params, 'CubicSpline', threads=threads)
    s.a_eval.count_pairs = True
    s.initialise()
    o.initialise()
    assert s.a_eval.last_pairs == o.pairs_last_eval > 0
    for _ in range(steps):
        assert abs(s.dt - o.dt) <= 1e-6 * o.dt
        s.step()
        o.step()
    assert s.a_eval.last_pairs == o.pairs_last_eval
    assert abs(s.dt - o.dt) <= 1e-6 * o.dt and abs(s.t - o.t) <= 1e-6 * o.t
    s.pull()
    _compare_state(pas, opas, params)
    return s.backend.stats()


def check_dam_break_2d_gate_vs_oracle(dx, steps, threads=4):
    """The 2-D gate case (WendlandQuintic, update_h, HG correction) under TVD-RK3."""
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_2d_particles(dx=dx)
    params = dict(geo.dam_break_2d_params(dx=dx), integrator='TVDRK3')
    assert params['update_h']
    opas = copy_arrays(pas)
    s = _solver(pas, params, 'WendlandQuintic')
    o = TVDRK3OracleSolver(opas, params, 'WendlandQuintic', threads=threads)
    s.a_eval.count_pairs = True
    for _ in range(steps):
        s.step()
        o.step()
        assert abs(s.dt - o.dt) <= 1e-6 * o.dt
    assert s.a_eval.last_pairs == o.pairs_last_eval
    s.pull()
    _compare_state(pas, opas, params)
    assert np.allclose(pas[0].h, opas[0].h, rtol=1e-7)


def check_dt_comes_from_the_third_evaluation(dx, device_dt):
    """After one step dt is the proposal of the THIRD evaluation's factors; the second
    evaluation's would differ by far more than the tolerance (random velocities)."""
    pas, params = _dam_break(dx, vscale=3.0)
    params['n_damp'] = 0
    opas = copy_arrays(pas)
    s = _solver(pas, params, device_dt=device_dt)
    o = TVDRK3OracleSolver(opas, params, 'CubicSpline', threads=4)
    s.initialise()
    o.initialise()
    proposals = []
    evaluate = o.compute_accelerations

    def compute_accelerations():
        evaluate()
        proposals.append(o._compute_timestep())
    o.compute_accelerations = compute_accelerations
    o.step()
    s.step()
    assert len(proposals) == 3 and o.dt == proposals[2]
    assert abs(proposals[1] - proposals[2]) > 1e-4 * proposals[2], proposals
    assert abs(s.dt - proposals[2]) <= 1e-6 * proposals[2], (s.dt, proposals)


# ---- 4. time control --------------------------------------------------------------------------
def check_device_dt_is_bitwise_host_dt(dx, steps):
    """Device-resident dt (three evaluations per step, the factors reduced by the fused stage3)
    and the host path give bitwise the same t, dt and trajectory, through the damped start and
    a tf-limited solve() that lands on tf."""
    out = {}
    for mode in (True, False):
        pas, params = _dam_break(dx, vscale=1.0)
        params['n_damp'] = 10
        s = _solver(pas, params, device_dt=mode)
        s.initialise()
        assert s.integrator.device_dt is mode
        for _ in range(steps):
            s.step()
        t1, dt1 = s.t, s.dt
        s.tf = t1 + 4.5 * dt1
        s.solve(1000)
        assert abs(s.tf - s.t) <= s._eps(), (s.tf, s.t)
        s.pull()
        out[mode] = (t1, dt1, s.count, s.t, s.dt,
                     [dict((k, pa.properties[k].copy()) for k in STATE) for pa in pas])
    a, b = out[True], out[False]
    assert a[:5] == b[:5], (a[:5], b[:5])
    assert a[2] == steps + 5
    for pa, pb_ in zip(a[5], b[5]):
        for k, v in pa.items():
            assert np.array_equal(v, pb_[k]), k


def check_post_stage_times(dx, steps=3):
    """Post-stage callbacks see (t + dt/3, 1), (t + 2dt/3, 2), (t + dt, 3), as in the reference."""
    pas, params = _dam_break(dx)
    s = _solver(pas, params)
    seen = []
    s.add_post_stage_callback(lambda t, dt, stage: seen.append((t, dt, stage)))
    s.initialise()
    for _ in range(steps):
        t, dt = s.t, s.dt
        del seen[:]
        s.step()
        assert seen == [(t + 1. / 3 * dt, dt, 1), (t + 2. / 3 * dt, dt, 2), (t + dt, dt, 3)], seen


def check_forced_repeats_change_nothing(dx, steps):
    """A deferred drift check that says "repeat" after the evaluation before stage 2, and one
    before stage 3: the repeat (plain update + evaluation) overwrites everything the first
    evaluation wrote, and the stages after it -- with their speculative records and, in
    stage 3, the dt factors -- run as without it.  The repeated evaluation packs its records
    through the light update instead of the fused stage kernel; its fp32 sums may round
    differently in the last bit (as under EPEC), so the runs agree to 1e-9 of h0 / c0 / rho0,
    a thousand times inside the oracle bars, with the same t and dt."""
    out = {}
    for forced in ((), (1, 2)):
        pas, params = _dam_break(dx, vscale=0.5)
        s = _solver(pas, params)
        s.initialise()
        nn, calls = s.nnps, [0]
        confirm = nn.confirm

        def forced_confirm():
            k = calls[0] % 3                 # 0, 1, 2: the evaluation before stage k + 1
            calls[0] += 1
            return confirm() or k in forced
        nn.confirm = forced_confirm
        for _ in range(steps):
            s.step()
        st = s.backend.stats()
        s.pull()
        assert calls[0] == 3 * steps
        out[forced] = (s.t, s.dt, pas, st, params)
    a, b = out[()], out[(1, 2)]
    assert b[3]['light_updates'] == a[3]['light_updates'] + 2 * steps   # the repeats really ran
    assert b[3]['full_builds'] == a[3]['full_builds']
    assert abs(a[0] - b[0]) <= 1e-12 * a[0] and abs(a[1] - b[1]) <= 1e-12 * a[1]
    _compare_state(b[2], a[2], a[4], pos=1e-9, vel=1e-9, rho=1e-9)


def check_restart_vs_oracle(tmp_path, dx, steps_before, steps_after):
    """Dump, restart a fresh solver from the file, and compare with the oracle restarted from
    the same file the same way (test_output.py's protocol, under TVD-RK3)."""
    from pysph_b200 import output
    import pysph_b200 as pb
    pas, params = _dam_break(dx)
    s = _solver(pas, params)
    for _ in range(steps_before):
        s.step()
    f = s.dump_output(str(tmp_path), 'rk3')
    sd = output.load(f)['solver_data']
    pas2, _ = _dam_break(dx)
    s2 = _solver(pas2, params)
    s2.load_output(f)
    data = output.load(f)
    opas = [data['arrays'][pa.name] for pa in pas]
    for q, pa in zip(opas, pas):
        for k in pa.properties:
            if k not in q.properties:
                q.add_property(k)
    o = TVDRK3OracleSolver(opas, dict(params), 'CubicSpline', threads=4)
    o.t, o.dt, o.count = float(sd['t']), float(sd['dt']), steps_before
    o.initialise()
    s2.initialise()
    assert abs(s2.dt - o.dt) <= 1e-6 * o.dt
    for _ in range(steps_after):
        s2.step()
        o.step()
    s2.pull()
    assert s2.count == steps_before + steps_after and abs(s2.t - o.t) <= 1e-6 * o.t
    _compare_state(pas2, opas, params)
    assert isinstance(s2.integrator, pb.TVDRK3Integrator)


# ---- 5. refusals ------------------------------------------------------------------------------
def check_refusals_on_the_library():
    """b200sph_stage keeps refusing which = 3; b200sph_stage_rk3 refuses which = 4; a periodic
    domain is refused under TVD-RK3 before anything runs; mirror planes are accepted."""
    import pysph_b200 as pb
    from pysph_b200._lib import B200Error
    pa = pb.get_particle_array_wcsph(name='f', x=np.linspace(0, 1, 8), h=np.full(8, 0.2))
    be = pb.B200Backend([pa])
    with pytest.raises(B200Error, match=r'which must be 0 \(initialize\), 1 \(stage1\) or 2 \(stage2\)'):
        be.ctx.call('b200sph_stage', -1, 3, 1e-3)
    with pytest.raises(B200Error, match='3 \\(stage3\\)'):
        be.ctx.call('b200sph_stage_rk3', -1, 4, 1e-3)
    with pytest.raises(B200Error, match='3 \\(stage3\\)'):
        be.ctx.call('b200sph_stage_rk3_dev', -1, -1)
    pas, params = _dam_break(0.1)
    with pytest.raises(NotImplementedError, match='periodic'):
        _solver(pas, params, domain=pb.DomainManager(xmin=0, xmax=1, periodic_in_x=True))
    pas, params = _dam_break(0.1)
    dom = pb.DomainManager(xmin=-0.1, xmax=3.5, ymin=-0.1, ymax=1.1, zmin=-0.1, zmax=1.1,
                           mirror_in_y=True)
    s = _solver(pas, params, domain=dom)
    assert isinstance(s.integrator, pb.TVDRK3Integrator)


# ---- the GPU tests ----------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _on_the_cuda_library(gpu_device):
    from pysph_b200 import _lib
    assert os.path.basename(_lib.LIB_PATH) == 'libb200sph.so', _lib.LIB_PATH


def test_tvdrk3_stepper_matches_reference_body():
    check_stepper_golden()


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_tvdrk3_fused_stage_is_bitwise_unfused(monkeypatch, records, device_dt):
    check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx=0.05)


def test_tvdrk3_dam_break_3d_vs_oracle():
    check_dam_break_3d_vs_oracle(dx=0.05, steps=25)


def test_tvdrk3_dam_break_3d_rebuilds_vs_oracle():
    st = check_dam_break_3d_vs_oracle(dx=0.05, steps=25, vscale=3.0)
    assert st['full_builds'] >= 2, st


def test_tvdrk3_dam_break_2d_gate_vs_oracle():
    check_dam_break_2d_gate_vs_oracle(dx=0.03, steps=25)


@pytest.mark.parametrize('device_dt', [True, False])
def test_tvdrk3_dt_from_the_third_evaluation(device_dt):
    check_dt_comes_from_the_third_evaluation(dx=0.05, device_dt=device_dt)


def test_tvdrk3_device_dt_is_bitwise_host_dt():
    check_device_dt_is_bitwise_host_dt(dx=0.05, steps=25)


def test_tvdrk3_post_stage_times():
    check_post_stage_times(dx=0.05)


def test_tvdrk3_forced_repeats_change_nothing():
    check_forced_repeats_change_nothing(dx=0.05, steps=6)


def test_tvdrk3_restart_vs_oracle(tmp_path):
    check_restart_vs_oracle(tmp_path, dx=0.05, steps_before=10, steps_after=8)


def test_tvdrk3_refusals_on_the_library():
    check_refusals_on_the_library()


# ---- slabs: 2 GPUs ----------------------------------------------------------------------------
def _slab_worker(rank, world, port, q, dx, steps):
    import torch
    import torch.distributed as dist
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from pysph_b200.parallel import make_slab_solver
    import test_gpu_multi as M
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    try:
        params = dict(geo.dam_break_3d_params(dx), integrator='TVDRK3')
        solver, pm, pas = make_slab_solver(dx, params, pb.CubicSpline(dim=3), rank, world,
                                           device=rank, n_damp=0)
        M._perturb(pas)
        solver.backend.push_all()
        solver.backend.use_torch_stream()
        for _ in range(steps):
            solver.step()
        t = solver.t
        solver.pull()
        q.put((rank, M._collect(pas), pm.n_full, pm.n_refresh, t))
    finally:
        dist.destroy_process_group()


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpus() < 2, reason='needs >= 2 GPUs')
def test_tvdrk3_slabs_match_one_gpu():
    """The slab decomposition under TVD-RK3 (adaptive dt, migration across the cuts) equals
    the one-GPU run by gid."""
    import socket
    import torch.multiprocessing as mp
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    import test_gpu_multi as M
    dx, steps, world = 0.04, 20, 2
    params = dict(geo.dam_break_3d_params(dx), integrator='TVDRK3', n_damp=0)
    pas = geo.dam_break_3d_particles(dx=dx)
    M._perturb(pas)
    s = _solver(pas, params)
    for _ in range(steps):
        s.step()
    t_ref = s.t
    s.pull()
    ref = M._collect(pas)
    sock = socket.socket()
    sock.bind(('127.0.0.1', 0))
    port = sock.getsockname()[1]
    sock.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_slab_worker, args=(r, world, port, q, dx, steps))
             for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    compare_slabs(out, ref, t_ref, params)


def compare_slabs(out, ref, t_ref, params, tol=5e-6):
    assert min(o[3] for o in out) > 0 and min(o[2] for o in out) >= 1
    for o in out:
        assert abs(o[4] - t_ref) <= 1e-6 * t_ref
    h0, c0 = params['h0'], params['c0']
    for name in ref:
        g_all = np.concatenate([o[1][name]['gid'] for o in out])
        assert np.array_equal(np.sort(g_all), np.sort(ref[name]['gid'])), name
        order_ref, order = np.argsort(ref[name]['gid']), np.argsort(g_all)
        for k, t in (('x', tol * h0), ('y', tol * h0), ('z', tol * h0), ('u', tol * c0),
                     ('v', tol * c0), ('w', tol * c0), ('rho', 5e-4)):
            a = np.concatenate([o[1][name][k] for o in out])[order]
            assert np.max(np.abs(a - ref[name][k][order_ref])) <= t, (name, k)
