"""The deferred initialize and the pool side of the EOS in the fused stage kernels.

On the fast path WCSPHStep.initialize (and WCSPHTVDRK3Step's, the same copy) launches nothing:
the next fused stage kernel copies x .. rho into x0 .. rho0 as it goes, and it also applies the
last evaluation's EOS calls to the pool's rho / p / cs, which the pair pass no longer does in a
launch of its own.  Everything the host can observe must stay what the separate kernels
(B200SPH_FUSE=0) give, bitwise: the state after whole runs, for both integrators, host and
device dt, 32- and 48-byte records, through list rebuilds and a forced repeat of an evaluation,
and every property pulled between the first evaluation and stage 1 and between steps (those
pulls run the deferred work first, so a run with them takes the other path through the code).
Wall particles start below rho0, so that TaitEOSHGCorrection clamps.

The check_* functions take the sizes as arguments: tests/test_deferred_init_on_cpu.py runs the
same checks, smaller, on the library emulation.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

OBSERVED = ('x0', 'y0', 'z0', 'u0', 'v0', 'w0', 'rho0', 'rho', 'p', 'cs')


def _dam_break(dx, integrator, vscale, seed=9):
    """The 3-D dam break with random fluid velocities (vscale > 0 uses up the list skin) and
    walls 0.5 % below rho0 (the HG correction clamps them at every evaluation)."""
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    rs = np.random.RandomState(seed)
    f = pas[0]
    for k in ('u', 'v', 'w'):
        f.properties[k][:] = rs.normal(scale=vscale, size=f.u.size)
    f.rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, f.u.size)
    for pa in pas[1:]:
        pa.rho[:] *= 1 - 0.005 * rs.uniform(0, 1, pa.rho.size)
    params = geo.dam_break_3d_params(dx)
    params['integrator'] = integrator
    params['n_damp'] = 6
    return pas, params


def _solver(pas, params, **kw):
    import pysph_b200 as pb
    keep = ('fluids', 'solids', 'dim', 'rho0', 'c0', 'h0', 'hdx', 'gamma', 'gx', 'gy', 'gz',
            'alpha', 'beta', 'tensile_correction', 'hg_correction', 'update_h',
            'summation_density', 'dt0', 'n_damp', 'cfl', 'integrator')
    p = dict((k, v) for k, v in params.items() if k in keep)
    return pb.make_wcsph_solver(pas, p, pb.CubicSpline(dim=params['dim']), **kw)


def _observed(pas):
    return [dict((k, pa.properties[k].copy()) for k in OBSERVED) for pa in pas]


def _run(monkeypatch, fuse, integrator, device_dt, dx, steps, vscale, pulls, forced=()):
    """steps of the dam break with B200SPH_FUSE=fuse; pulls: pull everything between the
    first evaluation and stage 1, and after every step; forced: the evaluations (counted from
    0, before stage k + 1) whose deferred drift check is made to say "repeat"."""
    monkeypatch.setenv('B200SPH_FUSE', fuse)
    pas, params = _dam_break(dx, integrator, vscale)
    s = _solver(pas, params, device_dt=device_dt)
    s.initialise()
    seen = []
    if pulls:
        stage1 = s.integrator.stage1

        def pulled_stage1():
            s.pull()
            seen.append(_observed(pas))
            stage1()
        s.integrator.stage1 = pulled_stage1
    if forced:
        nn, calls = s.nnps, [0]
        confirm = nn.confirm
        per_step = 3 if integrator == 'TVDRK3' else 2

        def forced_confirm():
            k = calls[0] % per_step
            calls[0] += 1
            return confirm() or k in forced
        nn.confirm = forced_confirm
    for _ in range(steps):
        s.step()
        if pulls:
            s.pull()
            seen.append(_observed(pas))
    st = s.backend.stats()
    s.pull()
    state = [dict((k, v.copy()) for k, v in pa.properties.items()) for pa in pas]
    return (s.t, s.dt, st['full_builds']), state, seen, st


def _assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0])
    for x, y in zip(a[1], b[1]):
        for k, v in x.items():
            assert np.array_equal(v, y[k]), k
    assert len(a[2]) == len(b[2])
    for i, (x, y) in enumerate(zip(a[2], b[2])):
        for pa_x, pa_y in zip(x, y):
            for k, v in pa_x.items():
                assert np.array_equal(v, pa_y[k]), (i, k)


def check_bitwise_the_separate_kernels(monkeypatch, integrator, records, device_dt, pulls, dx, steps):
    if records == '48':
        monkeypatch.setenv('B200SPH_RECORDS', '48')
    else:
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    new = _run(monkeypatch, '1', integrator, device_dt, dx, steps, 3.0, pulls)
    old = _run(monkeypatch, '0', integrator, device_dt, dx, steps, 3.0, pulls)
    st = new[3]
    assert st['full_builds'] >= 2, st                                  # lists were rebuilt
    assert st['fused_stages'] >= (2 if integrator == 'EPEC' else 3) * steps // 2, st
    assert (st['pair_launches_r32'] > 0) == (records == '32'), st
    _assert_same(new, old)


def check_forced_repeat_bitwise_the_separate_kernels(monkeypatch, integrator, dx, steps):
    """A repeated first evaluation (the pending initialize and the pool-side EOS meet a full
    rebuild and a second set of EOS calls) and a repeated last one."""
    monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    last = 2 if integrator == 'TVDRK3' else 1
    new = _run(monkeypatch, '1', integrator, False, dx, steps, 0.5, False, forced=(0, last))
    old = _run(monkeypatch, '0', integrator, False, dx, steps, 0.5, False, forced=(0, last))
    assert new[3]['fused_stages'] > 0
    _assert_same(new, old)


def check_epec_step_launches(monkeypatch, dx, steps=8):
    """A steady EPEC step (the lists reused, 32-byte records, host dt) launches the two pair
    kernels, the two fused stage kernels and k_dt_advance: no initialize, no k_eos_tab."""
    monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    monkeypatch.setenv('B200SPH_FUSE', '1')
    pas, params = _dam_break(dx, 'EPEC', 0.0)
    s = _solver(pas, params)
    s.initialise()
    s.step()
    steady = []
    a = s.backend.stats()
    for _ in range(steps):
        s.step()
        b = s.backend.stats()
        if b['full_builds'] == a['full_builds'] and b['fused_stages'] - a['fused_stages'] == 2:
            steady.append(b['kernel_launches'] - a['kernel_launches'])
        a = b
    assert len(steady) >= steps // 2 and set(steady) == {5}, steady


# ---- the GPU tests ----------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _on_the_cuda_library(gpu_device):
    from pysph_b200 import _lib
    assert os.path.basename(_lib.LIB_PATH) == 'libb200sph.so', _lib.LIB_PATH


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_deferred_init_is_bitwise_the_separate_kernels(monkeypatch, integrator, records, device_dt):
    check_bitwise_the_separate_kernels(monkeypatch, integrator, records, device_dt, False, dx=0.05, steps=20)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('records', ['32', '48'])
def test_pulls_between_evaluation_and_stage_see_the_separate_kernels(monkeypatch, integrator, records):
    check_bitwise_the_separate_kernels(monkeypatch, integrator, records, True, True, dx=0.05, steps=8)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_forced_repeat_is_bitwise_the_separate_kernels(monkeypatch, integrator):
    check_forced_repeat_bitwise_the_separate_kernels(monkeypatch, integrator, dx=0.05, steps=6)


def test_epec_step_launches(monkeypatch):
    check_epec_step_launches(monkeypatch, dx=0.05)
