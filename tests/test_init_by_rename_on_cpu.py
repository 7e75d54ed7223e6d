"""tests/test_gpu_init_by_rename.py on the library emulation (the loader of
test_library_on_cpu.py), smaller, where no GPU is available."""
import pytest

import test_gpu_init_by_rename as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

DX = 0.08


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('device_dt', [True, False])
@pytest.mark.parametrize('points', [t.EARLY, t.LATE], ids=['early', 'late'])
def test_pulled_state_is_bitwise_the_separate_kernels_emulated(emulated_library, monkeypatch, integrator,
                                                               device_dt, points):
    t.check_observed_state(monkeypatch, integrator, device_dt, points, dx=DX, steps=7)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_rebuild_and_repeat_between_the_stages_emulated(emulated_library, monkeypatch, integrator):
    t.check_rebuild_and_repeat_between_the_stages(monkeypatch, integrator, dx=DX, steps=3)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_the_buffers_change_names_only_without_ghosts_emulated(emulated_library, monkeypatch, integrator):
    t.check_the_buffers_change_names(monkeypatch, integrator, dx=DX)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('mid_step', [False, True])
def test_dump_and_restart_with_exchanged_buffers_emulated(emulated_library, monkeypatch, tmp_path, integrator,
                                                          mid_step):
    t.check_dump_and_restart(monkeypatch, tmp_path, integrator, DX, 3, 2, mid_step)
