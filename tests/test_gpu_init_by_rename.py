"""The deferred initialize taken by renaming the buffers.

Stage 1 of the fused stage kernels, in a context without ghosts, does not copy x .. rho into
x0 .. rho0: the library exchanges which buffers go by the two sets of names and the kernel
writes the stepped state into the buffers that have become x .. rho.  Nothing the host can
observe may tell: every property pulled after the initialize, between the first evaluation and
stage 1, between the stages and after the step is bitwise what the separate kernels
(B200SPH_FUSE=0) give, for both integrators, host and device dt, through a push of the
positions between the stages (a forced list rebuild) and a forced repeat of the evaluation
between the stages; so are a dump taken after an odd number of steps, one taken from a
post-stage callback in the middle of a step, and the runs restarted from them.  A context with
ghosts keeps the copy, and stays bitwise the separate kernels too.

The check_* functions take the sizes as arguments: tests/test_init_by_rename_on_cpu.py runs the
same checks, smaller, on the library emulation.
"""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_deferred_init import _dam_break, _solver

pytestmark = pytest.mark.gpu

EARLY = ('initialize', 'evaluation1')    # pulls that run the pending initialize as a copy
LATE = ('stage1', 'evaluation2', 'step')   # pulls that see the renamed buffers


def _everything(pas):
    return [dict((k, v.copy()) for k, v in pa.properties.items()) for pa in pas]


def _x_pointer(s):
    p = C.c_void_p()
    s.backend.ctx.call('b200sph_device_ptr', 0, 0, C.byref(p))
    return p.value


def _run(monkeypatch, fuse, integrator, device_dt, dx, steps, points, vscale=3.0, push_x=False,
         forced=(), ghosts=0):
    """steps of the dam break with B200SPH_FUSE=fuse, everything pulled at `points`;
    push_x: the positions pulled after stage 1 are pushed back and the kernel is set again (the
    next update rebuilds the lists); forced: the evaluations (counted from 0 within a step) whose deferred drift check
    is made to say "repeat"; ghosts: that many particles at the end of the largest wall array are ghosts."""
    monkeypatch.setenv('B200SPH_FUSE', fuse)
    monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    pas, params = _dam_break(dx, integrator, vscale)
    if ghosts:
        wall = max(pas[1:], key=lambda pa: pa.get_number_of_particles())
        wall.set_num_real_particles(wall.get_number_of_particles() - ghosts)
    import pysph_b200 as pb
    kernel = pb.CubicSpline(dim=params['dim'])
    s = _solver(pas, params, device_dt=device_dt)
    s.initialise()
    seen, evals, it = [], [0], s.integrator

    def observe():
        s.pull()
        seen.append(_everything(pas))

    def after(name, point, extra=None):
        fn = getattr(it, name)

        def wrapped(*a, **kw):
            fn(*a, **kw)
            if extra:
                extra()
            if point() in points:
                observe()
        setattr(it, name, wrapped)

    def evaluation():
        evals[0] += 1
        return 'evaluation%d' % evals[0]

    def pushed():
        if push_x:
            s.pull(['x'])
            s.backend.push(0, ['x'])
            s.nnps.set_kernel(kernel)
    after('initialize', lambda: 'initialize')
    after('compute_accelerations', evaluation)
    after('stage1', lambda: 'stage1', pushed)
    if forced:
        nn, calls = s.nnps, [0]
        confirm = nn.confirm
        per_step = 3 if integrator == 'TVDRK3' else 2

        def forced_confirm():
            k = calls[0] % per_step
            calls[0] += 1
            return confirm() or k in forced
        nn.confirm = forced_confirm
    pointers = []
    for _ in range(steps):
        evals[0] = 0
        s.step()
        if 'step' in points:
            observe()
        if 'pointer' in points:
            pointers.append(_x_pointer(s))
    st = s.backend.stats()
    s.pull()
    return (s.t, s.dt, st['full_builds']), _everything(pas), seen, st, pointers


def _assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0])
    assert len(a[2]) == len(b[2])
    for i, (x, y) in enumerate([(a[1], b[1])] + list(zip(a[2], b[2]))):
        for pa_x, pa_y in zip(x, y):
            assert sorted(pa_x) == sorted(pa_y)
            for k, v in pa_x.items():
                assert np.array_equal(v, pa_y[k]), (i - 1, k)


def check_observed_state(monkeypatch, integrator, device_dt, points, dx, steps):
    new = _run(monkeypatch, '1', integrator, device_dt, dx, steps, points)
    old = _run(monkeypatch, '0', integrator, device_dt, dx, steps, points)
    st = new[3]
    assert st['full_builds'] >= 2 and st['fused_stages'] >= steps, st
    assert len(new[2]) == len(points) * steps
    _assert_same(new, old)


def check_rebuild_and_repeat_between_the_stages(monkeypatch, integrator, dx, steps):
    kw = dict(vscale=0.5, push_x=True, forced=(1,))
    new = _run(monkeypatch, '1', integrator, False, dx, steps, LATE, **kw)
    old = _run(monkeypatch, '0', integrator, False, dx, steps, LATE, **kw)
    assert new[3]['full_builds'] >= steps and new[3]['fused_stages'] > 0, new[3]
    _assert_same(new, old)


def check_the_buffers_change_names(monkeypatch, integrator, dx, steps=5):
    """Without ghosts a fused stage 1 exchanges the buffers (x is found at one of two addresses,
    the other one after most steps); with ghosts it copies, and x stays where it is.  Either way the
    state is bitwise the separate kernels'."""
    for ghosts in (0, 40):
        new = _run(monkeypatch, '1', integrator, False, dx, steps, ('pointer',), 0.0, ghosts=ghosts)
        old = _run(monkeypatch, '0', integrator, False, dx, steps, ('pointer',), 0.0, ghosts=ghosts)
        assert new[3]['fused_stages'] >= 2 * (steps - 1), new[3]
        assert len(set(old[4])) == 1
        p = new[4]
        if ghosts:
            assert len(set(p)) == 1, p
        else:
            assert len(set(p)) == 2 and sum(p[i] != p[i + 1] for i in range(steps - 1)) >= steps // 2, p
        _assert_same(new, old)


def check_dump_and_restart(monkeypatch, tmp_path, integrator, dx, steps_before, steps_after, mid_step):
    """A dump after steps_before steps (odd: the buffers are exchanged), or one taken by a
    post-stage callback after stage 1 of the following step, and the run restarted from it."""
    from pysph_b200 import output
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
        d = str(tmp_path / ('fuse' + fuse))
        pas, params = _dam_break(dx, integrator, 0.5)
        s = _solver(pas, params)
        files = []
        if mid_step:
            def dump(t, dt, stage):
                if stage == 1 and s.count == steps_before:
                    files.append(s.dump_output(d, 'mid', detailed_output=True))
            s.add_post_stage_callback(dump)
        for _ in range(steps_before + (1 if mid_step else 0)):
            s.step()
        if not mid_step:
            files.append(s.dump_output(d, 'odd', detailed_output=True))
        assert len(files) == 1 and (s.backend.stats()['fused_stages'] > 0) == (fuse == '1')
        data = output.load(files[0])
        pas2, _ = _dam_break(dx, integrator, 0.5)
        s2 = _solver(pas2, params)
        s2.load_output(files[0])
        for _ in range(steps_after):
            s2.step()
        s2.pull()
        s.pull()
        out[fuse] = ((s2.t, s2.dt, s2.count), _everything(pas2),
                     [[dict(data['arrays'][pa.name].properties) for pa in pas], _everything(pas)])
    _assert_same(out['1'], out['0'])


# ---- the GPU tests ----------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _on_the_cuda_library(gpu_device):
    from pysph_b200 import _lib
    assert os.path.basename(_lib.LIB_PATH) == 'libb200sph.so', _lib.LIB_PATH


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('device_dt', [True, False])
@pytest.mark.parametrize('points', [EARLY, LATE], ids=['early', 'late'])
def test_pulled_state_is_bitwise_the_separate_kernels(monkeypatch, integrator, device_dt, points):
    check_observed_state(monkeypatch, integrator, device_dt, points, dx=0.05, steps=9)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_rebuild_and_repeat_between_the_stages(monkeypatch, integrator):
    check_rebuild_and_repeat_between_the_stages(monkeypatch, integrator, dx=0.05, steps=5)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_the_buffers_change_names_only_without_ghosts(monkeypatch, integrator):
    check_the_buffers_change_names(monkeypatch, integrator, dx=0.05)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('mid_step', [False, True])
def test_dump_and_restart_with_exchanged_buffers(monkeypatch, tmp_path, integrator, mid_step):
    check_dump_and_restart(monkeypatch, tmp_path, integrator, 0.05, 5, 4, mid_step)
