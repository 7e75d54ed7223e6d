"""tests/test_gpu_records32_eos_change.py on the library emulation (the loader of
test_library_on_cpu.py): a change of c0 or p0 between two 32-byte passes on one context, where
no GPU is available.  A module of its own: the emulation stays loaded until the module
that loaded it ends, so no GPU test may follow it in the same module."""
import pytest

import test_gpu_records32_eos_change as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


@pytest.mark.parametrize('stepped', [False, True], ids=['packed', 'fused_stage'])
@pytest.mark.parametrize('what', ['c0', 'p0'])
def test_records32_eos_change_vs_oracle_emulated(emulated_library, monkeypatch, what, stepped):
    t.check_eos_change(monkeypatch, what, stepped)
