"""tests/test_gpu_deferred_init.py on the library emulation (the loader of
test_library_on_cpu.py), smaller, where no GPU is available."""
import pytest

import test_gpu_deferred_init as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

DX = 0.08


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_deferred_init_is_bitwise_the_separate_kernels_emulated(emulated_library, monkeypatch, integrator, records,
                                                                device_dt):
    t.check_bitwise_the_separate_kernels(monkeypatch, integrator, records, device_dt, False, dx=DX, steps=16)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_pulls_between_evaluation_and_stage_emulated(emulated_library, monkeypatch, integrator):
    t.check_bitwise_the_separate_kernels(monkeypatch, integrator, '32', True, True, dx=DX, steps=6)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_forced_repeat_emulated(emulated_library, monkeypatch, integrator):
    t.check_forced_repeat_bitwise_the_separate_kernels(monkeypatch, integrator, dx=DX, steps=4)


def test_epec_step_launches_emulated(emulated_library, monkeypatch):
    t.check_epec_step_launches(monkeypatch, dx=DX)
