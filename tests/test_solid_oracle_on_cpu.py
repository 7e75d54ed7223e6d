"""tests/test_gpu_solid_oracle.py on the library emulation (the loader of test_library_on_cpu.py):
the elastic-dynamics passes and SolidMechStep against the fp64 oracle where no GPU is available.
A module of its own: the emulation stays loaded until the module that loaded it ends, so no GPU
test may follow it in the same module.  Also the oracle's own eigen_sym3 against numpy's fp64
eigh on the stress states of those tests."""
import numpy as np
import pytest

import test_gpu_solid_oracle as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

@pytest.mark.parametrize('split', [False, True], ids=['passes3', 'passes1then2'])
@pytest.mark.parametrize('kname,dim,grad3d', t.MATRIX)
def test_solid_pass_vs_oracle_emulated(emulated_library, kname, dim, grad3d, split):
    t.check_pass(kname, dim, grad3d, split=split)


def test_solid_pass_2d_full_stress_vs_oracle_emulated(emulated_library):
    t.check_pass('CubicSpline', 2, 0, full3x3=True)


@pytest.mark.parametrize('ghost_group1', [0, 1])
@pytest.mark.parametrize('kname,dim', t.KERNEL_DIMS)
def test_solid_ghosts_vs_oracle_emulated(emulated_library, kname, dim, ghost_group1):
    t.check_ghosts(kname, dim, ghost_group1)


@pytest.mark.parametrize('devdt', [False, True], ids=['dt', 'dev'])
@pytest.mark.parametrize('arr', [-1, 0])
def test_solid_stage_vs_oracle_emulated(emulated_library, arr, devdt):
    t.check_stage('CubicSpline', 3, arr, devdt)


def _projector_part(lam, V, positive):
    """sum over the eigenvalues > 0 (or all) of lam v v^T: unique even where eigenvalues
    repeat, unlike the eigenvector columns"""
    keep = lam > 0 if positive else np.ones(3, bool)
    return (V[:, keep] * lam[keep]) @ V[:, keep].T


@pytest.mark.parametrize('planar', [False, True])
@pytest.mark.parametrize('state', t.STATES)
def test_oracle_eigen_sym3_vs_numpy(state, planar):
    """orc_eigen_sym3 (the fp64 cyclic Jacobi behind the oracle's MonaghanArtificialStress):
    orthonormal eigenvectors, the reconstruction V diag(d) V^T = S and the positive spectral
    part sum_{d > 0} d v v^T -- what r is made of -- against numpy's eigh, per stress state"""
    from oracle import oracle as orc
    rs = np.random.RandomState(3)
    for _ in range(20):
        S, lam = t.stress_state(state, t.STRESS_A * rs.uniform(0.5, 2.0), rs, planar)
        d, V = orc.eigen_sym3(S)
        wl, wv = np.linalg.eigh(S)
        scale = max(np.max(np.abs(S)), 1e-300)
        assert np.max(np.abs(V.T @ V - np.eye(3))) <= 1e-14, state
        assert np.max(np.abs(_projector_part(d, V, False) - S)) <= 1e-14 * scale, state
        assert np.max(np.abs(np.sort(d) - wl)) <= 1e-14 * scale, state
        want = _projector_part(wl, wv, True)
        got = _projector_part(d, V, True)
        if state in ('zero', 'iso_compression'):
            assert np.all(got == 0.0), state
            continue
        # the eigenvalues of S are known to ~1e-16 max|S|: near zero (straddle_zero) the
        # positive part is as exact as the tiny eigenvalues' own rounding
        wscale = max(np.max(np.abs(want)), 1e-300)
        tol = t.R_TOL if state in ('straddle_zero', 'range_1e8') else 1e-13
        assert np.max(np.abs(got - want)) <= tol * wscale, (state, np.max(np.abs(got - want)) / wscale)
