"""tests/test_gpu_half_step_deferred.py on the library emulation (the loader of
test_library_on_cpu.py), smaller, where no GPU is available."""
import pytest

import test_gpu_half_step_deferred as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

DX = 0.08


@pytest.mark.parametrize('device_dt', [True, False])
@pytest.mark.parametrize('point', ['stage1', 'evaluation2'])
def test_pulled_between_the_stages_emulated(emulated_library, monkeypatch, device_dt, point):
    t.check_pulled_between_the_stages(monkeypatch, device_dt, point, dx=DX, steps=6)


@pytest.mark.parametrize('device_dt', [True, False])
def test_nothing_observed_forms_nothing_emulated(emulated_library, monkeypatch, device_dt):
    t.check_nothing_observed(monkeypatch, device_dt, dx=DX, steps=5)


def test_rebuilds_before_the_second_evaluation_emulated(emulated_library, monkeypatch):
    t.check_rebuilds_before_the_second_evaluation(monkeypatch, dx=DX, steps=8)


def test_forced_repeat_of_the_second_evaluation_emulated(emulated_library, monkeypatch):
    t.check_forced_repeat_of_the_second_evaluation(monkeypatch, dx=DX, steps=3)


def test_old_paths_leave_nothing_pending_emulated(emulated_library, monkeypatch):
    t.check_old_paths_leave_nothing_pending(monkeypatch, dx=DX, steps=3)


def test_dump_between_evaluation_and_stage_emulated(emulated_library, monkeypatch, tmp_path):
    t.check_dump_between_evaluation_and_stage(monkeypatch, tmp_path, DX, 2, 2)
