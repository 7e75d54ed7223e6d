"""The Interpolator without a GPU: the fp64 oracle against the reference's own bodies, the grid
helpers against the reference test's known answers, the Python refusals, and
tests/test_gpu_interpolator.py on the library emulation (the loader of test_library_on_cpu.py),
smaller."""
import numpy as np
import pytest

import test_gpu_interpolator as t
from helpers import load_golden
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


# ---- the oracle --------------------------------------------------------------------------------
def test_oracle_matches_goldens():
    """tests/interpolator_oracle.py against the reference's bodies, to 1e-12 of each case's
    largest value (order1: where its moment matrix is not singular to rounding)."""
    from interpolator_oracle import interpolate
    for c in load_golden('interpolator_cases.json'):
        for m in t.METHODS:
            want = np.array(c['results'][m])
            got = interpolate(c, m)
            if m == 'order1':
                got, cond, _ = got
                keep = np.repeat(cond < 1e12, 4)
                assert np.all(got[np.repeat(np.isinf(cond), 4)] == 0.0)
                got, want = got[keep], want[keep]
            scale = max(np.max(np.abs(want)), 1e-300)
            assert np.max(np.abs(got - want)) <= 1e-12 * scale, (c['kernel'], c['dim'], c['periodic'], m)


def test_goldens_cover_the_edges():
    """every method, kernel and dimension; periodic boxes with probes outside them; probes with
    no neighbour (zero weight); gj_solve's early return on a collinear neighbourhood"""
    from interpolator_oracle import interpolate
    cases = load_golden('interpolator_cases.json')
    assert set((c['kernel'], c['dim']) for c in cases) == set(
        (k, d) for k in ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian') for d in (1, 2, 3)
        if (k, d) != ('WendlandQuintic', 1))
    assert all(set(c['results']) == set(t.METHODS) for c in cases)
    assert any(c['periodic'] for c in cases)
    for c in cases:
        assert 'f' not in c['arrays']['solid'] and len(set(c['arrays']['fluid']['h'])) > 1
        if c['periodic']:
            px, box = np.array(c['probes']['x']), c['box']
            assert np.any(px < box['lo'][0]) and np.any(px > box['hi'][0])
        else:
            assert c['results']['shepard'][-2 if c['dim'] != 2 else -3] == 0.0   # no neighbour
        if c['dim'] == 2 and not c['periodic']:
            _, cond, _ = interpolate(c, 'order1')
            assert np.isinf(cond[-1]) and c['results']['order1'][-4:] == [0.0] * 4


# ---- the grid helpers (the reference's TestGetNxNyNz) ----------------------------------------------
def test_get_nx_ny_nz():
    from pysph_b200 import get_nx_ny_nz
    assert list(get_nx_ny_nz(100, (0.0, 1.5, 0.0, 0.0, 0.0, 0.0))) == [100, 1, 1]
    assert list(get_nx_ny_nz(100, (0.0, 0.0, 0.0, 1.123, 0.0, 0.0))) == [1, 100, 1]
    assert list(get_nx_ny_nz(100, (0.0, 0.0, 0.0, 0.0, 0.0, 3.0))) == [1, 1, 100]
    assert list(get_nx_ny_nz(100, (0.0, 1.0, 0.5, 1.5, 0.0, 0.0))) == [10, 10, 1]
    assert list(get_nx_ny_nz(100, (0.0, 0.0, 0, 1, 0.5, 1.5))) == [1, 10, 10]
    assert list(get_nx_ny_nz(1000, (0.0, 1.0, 0.5, 1.5, -1.0, 0.0))) == [10, 10, 10]
    assert list(get_nx_ny_nz(1000, (0.0, 1.0, 0.5, 1.5, -1.0, 2.0))) == [7, 7, 21]


def test_get_bounding_box():
    import pysph_b200 as pb
    a = pb.get_particle_array(name='a', x=np.array([0.0, 1.0]), y=np.array([0.0, 2.0]), z=np.zeros(2))
    b = pb.get_particle_array(name='b', x=np.array([-1.0]), y=np.array([1.0]), z=np.array([4.0]))
    assert np.allclose(pb.get_bounding_box([a, b], tight=True), [-1, 1, 0, 2, 0, 4])
    assert np.allclose(pb.get_bounding_box([a, b]), [-1.1, 1.1, -0.1, 2.1, -0.2, 4.2])


def test_python_refusals():
    """(before any device work)"""
    import pysph_b200 as pb
    pa = pb.get_particle_array(name='a', x=np.linspace(0, 1, 5), y=np.linspace(0, 1, 5), z=np.zeros(5),
                               h=np.full(5, 0.1))
    with pytest.raises(NotImplementedError, match='equations'):
        pb.Interpolator([pa], num_points=10, equations=[])
    with pytest.raises(RuntimeError, match='not implemented'):
        pb.Interpolator([pa], num_points=10, method='order2')
    with pytest.raises(NotImplementedError, match='order1 with a 3-D kernel'):
        pb.Interpolator([pa], num_points=10, method='order1', kernel=pb.Gaussian(dim=3))


# ---- the GPU checks on the library emulation -----------------------------------------------------
@pytest.mark.parametrize('idx', list(range(15)))
def test_fixture_emulated(emulated_library, idx):
    t.check_fixture(idx)


def test_reference_cases_emulated(emulated_library):
    t.check_reference_cases(n=101, num_points=1000)


@pytest.mark.parametrize('integrator', ['EPEC', 'TVDRK3'])
def test_live_vs_private_emulated(emulated_library, integrator):
    t.check_live_vs_private(0.1, integrator, steps=5)


def test_run_untouched_emulated(emulated_library):
    t.check_run_untouched(0.1, steps=8)


def test_periodic_edac_emulated(emulated_library):
    t.check_periodic_edac(16, steps=3)


def test_refusals_emulated(emulated_library):
    t.check_refusals()
