"""The half step a fused stage 1 leaves pending.

In a context without ghosts, the fused WCSPHStep stage 1 that takes the initialize by renaming
does not store the predicted x .. rho, nor the p / cs of the EOS calls it applies to the pool:
stage 2 reads none of them but rho, which it forms again, and the second evaluation reads the
predicted state from the 32-byte records.  The pair pass of that evaluation writes into a spare
set of arho, au .. az so that the first
evaluation's accelerations stay readable, and whatever could observe the pending values forms
them first (half_materialise).  Every property pulled after stage 1, between the second
evaluation and stage 2, after a rebuild of the lists before the second evaluation and after a
forced repeat of it must be bitwise what the separate kernels (B200SPH_FUSE=0) give; so must a
dump taken between the second evaluation and stage 2, and a run restarted from it.  A step that
nothing observes forms nothing (stats()['half_materialised'] stays 0), and TVD-RK3 and a context
with ghosts never leave a half step pending.

The check_* functions take the sizes as arguments: tests/test_half_step_deferred_on_cpu.py runs
the same checks, smaller, on the library emulation.
"""
import os

import pytest

from test_gpu_deferred_init import _dam_break, _solver
from test_gpu_init_by_rename import _assert_same, _everything, _run

pytestmark = pytest.mark.gpu


def check_pulled_between_the_stages(monkeypatch, device_dt, point, dx, steps):
    """one pull per step after stage 1 or after the second evaluation: each forms the half step
    once (unless the rebuild of the lists before the second evaluation already did)"""
    new = _run(monkeypatch, '1', 'EPEC', device_dt, dx, steps, (point,))
    old = _run(monkeypatch, '0', 'EPEC', device_dt, dx, steps, (point,))
    st = new[3]
    assert st['fused_stages'] >= steps and 0 < st['half_materialised'] <= steps, st
    assert old[3]['half_materialised'] == 0
    _assert_same(new, old)


def check_nothing_observed(monkeypatch, device_dt, dx, steps):
    """no drift, no pull between the stages: no half step is ever formed"""
    new = _run(monkeypatch, '1', 'EPEC', device_dt, dx, steps, ('step',), vscale=0.0)
    old = _run(monkeypatch, '0', 'EPEC', device_dt, dx, steps, ('step',), vscale=0.0)
    st = new[3]
    assert st['fused_stages'] >= 2 * (steps - 1) and st['half_materialised'] == 0, st
    _assert_same(new, old)


def check_rebuilds_before_the_second_evaluation(monkeypatch, dx, steps):
    """a fast flow: the lists are rebuilt (proactively or after a failed check) between the stages"""
    new = _run(monkeypatch, '1', 'EPEC', True, dx, steps, ('evaluation2', 'step'), vscale=3.0)
    old = _run(monkeypatch, '0', 'EPEC', True, dx, steps, ('evaluation2', 'step'), vscale=3.0)
    st = new[3]
    assert st['full_builds'] >= 3 and st['half_materialised'] > 0, st
    _assert_same(new, old)


def check_forced_repeat_of_the_second_evaluation(monkeypatch, dx, steps):
    """the deferred check before every second evaluation says "repeat": that evaluation has
    already written into the spare accelerations, and the full build forms the half step from
    the first evaluation's set"""
    kw = dict(vscale=0.5, forced=(1,))
    new = _run(monkeypatch, '1', 'EPEC', False, dx, steps, ('step',), **kw)
    old = _run(monkeypatch, '0', 'EPEC', False, dx, steps, ('step',), **kw)
    st = new[3]
    assert st['half_materialised'] >= 1, st
    _assert_same(new, old)


def check_old_paths_leave_nothing_pending(monkeypatch, dx, steps):
    """TVD-RK3, and WCSPHStep with ghosts, store the whole stage: pulls form nothing"""
    for integrator, ghosts in (('TVDRK3', 0), ('EPEC', 40)):
        points = ('stage1', 'evaluation2')
        new = _run(monkeypatch, '1', integrator, False, dx, steps, points, ghosts=ghosts)
        old = _run(monkeypatch, '0', integrator, False, dx, steps, points, ghosts=ghosts)
        assert new[3]['fused_stages'] > 0 and new[3]['half_materialised'] == 0, new[3]
        _assert_same(new, old)


def check_dump_between_evaluation_and_stage(monkeypatch, tmp_path, dx, steps_before, steps_after):
    """a dump taken after the second evaluation of step steps_before + 1, and the run restarted
    from it"""
    from pysph_b200 import output
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
        d = str(tmp_path / ('fuse' + fuse))
        pas, params = _dam_break(dx, 'EPEC', 0.5)
        s = _solver(pas, params)
        it, evals, files = s.integrator, [0], []
        compute = it.compute_accelerations

        def compute_and_dump(*a, **kw):
            compute(*a, **kw)
            evals[0] += 1
            if evals[0] == 2 * steps_before + 2:
                files.append(s.dump_output(d, 'mid', detailed_output=True))
        it.compute_accelerations = compute_and_dump
        for _ in range(steps_before + 1):
            s.step()
        assert len(files) == 1
        if fuse == '1':
            assert s.backend.stats()['half_materialised'] >= 1
        data = output.load(files[0])
        pas2, _ = _dam_break(dx, 'EPEC', 0.5)
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


@pytest.mark.parametrize('device_dt', [True, False])
@pytest.mark.parametrize('point', ['stage1', 'evaluation2'])
def test_pulled_between_the_stages(monkeypatch, device_dt, point):
    check_pulled_between_the_stages(monkeypatch, device_dt, point, dx=0.05, steps=9)


@pytest.mark.parametrize('device_dt', [True, False])
def test_nothing_observed_forms_nothing(monkeypatch, device_dt):
    check_nothing_observed(monkeypatch, device_dt, dx=0.05, steps=8)


def test_rebuilds_before_the_second_evaluation(monkeypatch):
    check_rebuilds_before_the_second_evaluation(monkeypatch, dx=0.05, steps=14)


def test_forced_repeat_of_the_second_evaluation(monkeypatch):
    check_forced_repeat_of_the_second_evaluation(monkeypatch, dx=0.05, steps=5)


def test_old_paths_leave_nothing_pending(monkeypatch):
    check_old_paths_leave_nothing_pending(monkeypatch, dx=0.05, steps=5)


def test_dump_between_evaluation_and_stage(monkeypatch, tmp_path):
    check_dump_between_evaluation_and_stage(monkeypatch, tmp_path, 0.05, 4, 4)
