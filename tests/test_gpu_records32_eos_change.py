"""The 32-byte records carry p / rho^2, formed once per particle with the EOS constants rho0,
B = rho0 c0^2 / 7 and the pressure offset.  A pass whose EOS has another c0 or p0 than the one
the records were packed with must repack them: here the second of two passes on one context
changes c0 (or p0 of TaitEOS), with no push in between, and must still take the 32-byte
records and match the fp64 oracle.  The
stepped variant does the same after solver steps, so that the records the change meets were
written by the fused stage kernel (k_stage_pack).  Every test here runs on the GPU;
test_records32_eos_change_on_cpu.py runs the same checks on the library emulation."""
import os

import pytest

import test_gpu_records32_oracle as t
from helpers import copy_arrays

pytestmark = pytest.mark.gpu

KNAME, DIM = 'CubicSpline', 3


@pytest.fixture(autouse=True)
def _cuda_library(gpu_device):
    """these tests must reach libb200sph.so, not an emulation that another module loaded"""
    from pysph_b200 import _lib
    assert os.path.basename(_lib.load()._name) == 'libb200sph.so', _lib.load()._name


def _changed(eos, what):
    """the same EOS calls with c0 x 1.3, or with the offset p0 x 3 (the 'p0' calls: every
    array a plain TaitEOS)"""
    if what == 'c0':
        return [(hg, r, 1.3 * c, g, p0) for hg, r, c, g, p0 in eos]
    return [(hg, r, c, g, 3.0 * p0) for hg, r, c, g, p0 in eos]


def _pass_vs_oracle(s, pas, eos):
    opas = copy_arrays(pas)
    eqs = t._equations()
    pairs, r32 = t._device_pass(s, pas, eqs, eos, t.PROG)
    opairs = t._oracle_pass(opas, KNAME, DIM, eqs, eos, t.PROG)
    assert r32 == 1
    assert pairs == opairs > 0
    t._compare(pas, opas)


def check_eos_change(monkeypatch, what, stepped):
    pas, params = t._case(KNAME, DIM)
    s = t._solver(monkeypatch, KNAME, DIM, '32', pas, params)
    eos = t._eos_calls('hg' if what == 'c0' else 'p0')
    if stepped:
        for _ in range(3):
            s.step()
        assert s.backend.stats()['fused_stages'] > 0
        s.pull()
        # the solver's evaluation runs these before its pair passes
        s.backend.ctx.call('b200sph_update_domain')
        s.backend.ctx.call('b200sph_nnps_update')
    else:
        _pass_vs_oracle(s, pas, eos)
    _pass_vs_oracle(s, pas, _changed(eos, what))


@pytest.mark.parametrize('stepped', [False, True], ids=['packed', 'fused_stage'])
@pytest.mark.parametrize('what', ['c0', 'p0'])
def test_records32_eos_change_vs_oracle(gpu_device, monkeypatch, what, stepped):
    check_eos_change(monkeypatch, what, stepped)
