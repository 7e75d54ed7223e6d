"""tests/test_gpu_records32_oracle.py on the library emulation (the loader of
test_library_on_cpu.py): the 32-byte WCSPH pair kernel against the fp64 oracle for every
(kernel, dim), trajectories with kernels other than CubicSpline, and the choice of layout,
where no GPU is available.  A module of its own: the emulation stays loaded until the module
that loaded it ends, so no GPU test may follow it in the same module."""
import pytest

import test_gpu_records32_oracle as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('variant', ['hg', 'p0'])
@pytest.mark.parametrize('kname,dim', t.KERNEL_DIMS)
def test_pair_pass_vs_oracle_emulated(emulated_library, monkeypatch, kname, dim, variant,
                                      records):
    t.check_pass_vs_oracle(monkeypatch, kname, dim, variant, records)


@pytest.mark.parametrize('kname', ['WendlandQuintic', 'QuinticSpline'])
def test_trajectory_vs_oracle_emulated(emulated_library, kname):
    t.check_trajectory(kname)


@pytest.mark.parametrize('case', sorted(t.LAYOUT_CASES))
def test_layout_choice_vs_oracle_emulated(emulated_library, monkeypatch, case):
    t.check_layout(monkeypatch, case)
