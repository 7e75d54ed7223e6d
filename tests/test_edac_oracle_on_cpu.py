"""tests/test_gpu_edac_oracle.py on the library emulation (the loader of test_library_on_cpu.py):
the EDAC passes against the fp64 oracle for every (kernel, dim) and variant where no GPU is
available.  A module of its own: the emulation stays loaded until the module that loaded it
ends, so no GPU test may follow it in the same module."""
import pytest

import test_gpu_edac_oracle as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


@pytest.mark.parametrize('variant', sorted(t.VARIANTS))
@pytest.mark.parametrize('kname,dim', t.KERNEL_DIMS)
def test_tvf_pass_vs_oracle_emulated(emulated_library, kname, dim, variant):
    t.check_pass(kname, dim, variant)
