"""tests/test_gpu_neighbour_lists.py on the library emulation (the loader of
test_library_on_cpu.py): what the persistent neighbour lists hold, destination by destination,
against the fp64 brute force, while a build is reused to the limit of its skin, where no GPU is
available.  A module of its own: the emulation stays loaded until the module that loaded it
ends, so no GPU test may follow it in the same module."""
import pytest

import test_gpu_neighbour_lists as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_skin_shell_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_skin_shell(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_growing_and_unequal_h_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_growing_h(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_past_the_limit_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_past_the_limit(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,pattern,ncase,zorder', t.PERIODIC)
def test_periodic_emulated(emulated_library, monkeypatch, dim, pattern, ncase, zorder):
    t.check_periodic(monkeypatch, dim, pattern, ncase, zorder)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_crowds_tiles_and_capacity_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_crowds(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_capacity_regrows_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_capacity(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim', t.DIMS)
def test_all_in_one_cell_emulated(emulated_library, monkeypatch, dim):
    t.check_one_cell(monkeypatch, dim, 0)


@pytest.mark.parametrize('dim,zorder', t.ZORDER)
def test_two_groups_force_the_union_emulated(emulated_library, monkeypatch, dim, zorder):
    t.check_two_groups(monkeypatch, dim, zorder)


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('dim', [2, 3])
def test_pair_pass_counts_emulated(emulated_library, monkeypatch, dim, records):
    t.check_pair_pass(monkeypatch, dim, records)


@pytest.mark.parametrize('dim', [2, 3])
def test_tvf_pass_counts_emulated(emulated_library, monkeypatch, dim):
    t.check_tvf_pass(monkeypatch, dim)


@pytest.mark.parametrize('dim', [2, 3])
def test_solid_pass_counts_emulated(emulated_library, monkeypatch, dim):
    t.check_solid_pass(monkeypatch, dim)
