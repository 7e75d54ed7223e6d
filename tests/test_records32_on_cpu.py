"""tests/test_gpu_records32.py on the library emulation (the loader of test_library_on_cpu.py):
the host logic of the 32-byte records -- when they are chosen, when they are repacked -- and
their arithmetic, where no GPU is available.  Small dam breaks (dx = 0.08) keep it quick."""
import pytest

import test_gpu_records32 as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


def _call(fn, lib, **kw):
    fn = getattr(fn, '__wrapped__', fn)
    with pytest.MonkeyPatch.context() as mp:
        return fn(lib, mp, **kw)


def test_records32_match_records48_emulated(emulated_library):
    _call(t.test_records32_match_records48, emulated_library, dx=0.08, steps=12)


def test_records32_fused_stage_bitwise_emulated(emulated_library):
    _call(t.test_records32_fused_stage_is_bitwise_the_separate_kernels, emulated_library, dx=0.08, steps=8)


@pytest.mark.parametrize('edit', [t._perturb_h, t._perturb_m], ids=['h', 'm'])
def test_nonuniform_h_or_m_emulated(emulated_library, edit):
    _call(t.test_nonuniform_h_or_m_keeps_48_byte_records, emulated_library, edit=edit, steps=2)


def test_pushed_mass_is_noticed_emulated(emulated_library):
    _call(t.test_pushed_mass_is_noticed, emulated_library)


def test_ranged_group_takes_48_byte_records_emulated(emulated_library):
    _call(t.test_ranged_group_takes_48_byte_records, emulated_library)
