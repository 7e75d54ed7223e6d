"""TEST INFRASTRUCTURE: DensityCorrection's filters in fp64 numpy, and the oracle solvers with
the tool.

``density_filter`` restates ShepardFilter / MLSFirstOrder2D / MLSFirstOrder3D
(pysph/sph/wc/density_correction.py) with gj_solve (pysph/sph/wc/linalg.py:94-166) in its
operation order, vectorised over the destinations; the kernel values come from the fp64
oracle (oracle.kernel_w).  ``with_density_correction`` adds the tool's post_step
(pysph/solver/tools.py:200-207) to WCSPHOracleSolver or TVDRK3OracleSolver.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle import oracle as orc

NP = {'shepard': 0, 'mls2d_1': 3, 'mls3d_1': 4}


def _pairs(pos, h, k):
    """(i, j) with r^2 < (k h_i)^2 or r^2 < (k h_j)^2 (linked_list_nnps.pyx:188), sorted by i
    then j, the particle itself included"""
    tree = cKDTree(pos)
    pr = tree.query_pairs(k * float(np.max(h)) * (1 + 1e-9), output_type='ndarray')
    i = np.concatenate([pr[:, 0], pr[:, 1], np.arange(len(pos))])
    j = np.concatenate([pr[:, 1], pr[:, 0], np.arange(len(pos))])
    d = pos[i] - pos[j]
    r2 = np.sum(d * d, axis=1)
    ok = (r2 < (k * h[i]) ** 2) | (r2 < (k * h[j]) ** 2)
    i, j = i[ok], j[ok]
    o = np.lexsort((j, i))
    return i[o], j[o]


def gj_solve(m):
    """gj_solve on a stack of augmented matrices m[N, n, n + 1] (in place); returns the mask of
    the systems that did NOT take one of its early returns"""
    N, n = m.shape[0], m.shape[1]
    ok = np.ones(N, dtype=bool)
    with np.errstate(all='ignore'):
        for c in range(n):
            for r in range(c + 1, n):
                d = m[:, c, c].copy()
                ok &= ~(np.abs(d) < 1e-12)
                cc = -m[:, r, c] / d
                for j in range(n + 1):
                    m[:, r, j] = m[:, r, j] + cc * m[:, c, j]
        for rb in range(n - 1, -1, -1):
            zero = m[:, rb, rb] == 0
            ok &= ~(zero & (np.abs(m[:, rb, n]) > 1e-12))
            nz = ~zero
            for bc in range(n, rb - 1, -1):
                m[nz, rb, bc] = m[nz, rb, bc] / m[nz, rb, rb]
            for ku in range(rb - 1, -1, -1):
                for kl in range(n, rb - 1, -1):
                    kk = -m[nz, ku, rb] / m[nz, rb, rb]
                    m[nz, ku, kl] = m[nz, ku, kl] + kk * m[nz, rb, kl]
    return ok


def density_filter(pa, corr, kernel, dim):
    """One Group([Filter(pa, [pa])], real=False) on every particle of ``pa`` (in place):
    rhotmp = rho, then rho from rhotmp.  Returns rhotmp."""
    props = pa.properties
    n = pa.get_number_of_particles()
    pos = np.stack([props[c][:n] for c in 'xyz'], axis=1)
    h, m, rho = props['h'][:n], props['m'][:n], props['rho'][:n]
    rhotmp = rho.copy()
    if 'rhotmp' in props:
        props['rhotmp'][:n] = rhotmp
    k = orc.load().orc_kernel_radius_scale(orc.K_IDS[kernel])
    i, j = _pairs(pos, h, k)
    xij = pos[i] - pos[j]
    if corr == 'mls2d_1':
        xij[:, 2] = 0.0
    rij = np.sqrt(np.sum(xij * xij, axis=1))
    hij = (h[i] + h[j]) * 0.5
    w = np.array([orc.kernel_w(kernel, dim, r, hh) for r, hh in zip(rij, hij)])
    new = np.zeros(n)
    if corr == 'shepard':
        tmp = np.zeros(n)
        np.add.at(tmp, i, w * m[j] / rhotmp[j])
        np.add.at(new, i, w * m[j])
        new = new / tmp
    else:
        nn = NP[corr]
        p = np.concatenate([np.ones((len(i), 1)), xij[:, :nn - 1]], axis=1)
        aug = np.zeros((n, nn, nn + 1))
        for a in range(nn):
            for b in range(nn):
                np.add.at(aug[:, a, b], i, p[:, a] * p[:, b] * m[j] * w / rhotmp[j])
        aug[:, 0, nn] = 1.0
        ok = gj_solve(aug)
        res = np.zeros((n, nn))
        res[:, 0] = 1.0
        res[ok] = aug[ok, :, nn]
        b = res[i]
        np.add.at(new, i, m[j] * (np.sum(b * p, axis=1) * w))
    rho[:] = new
    return rhotmp


def with_density_correction(base):
    """``base`` (an oracle solver class) with DensityCorrection's post_step after every step,
    before t and dt advance (solver.py:480-491)."""

    class Solver(base):
        def __init__(self, particles, params, kernel='CubicSpline', threads=1, names=(),
                     corr='shepard', freq=10, filter_kernel=None):
            base.__init__(self, particles, params, kernel, threads=threads)
            self.names, self.corr, self.freq = list(names), corr, freq
            self.filter_kernel = filter_kernel or kernel
            self.tool_count = 1
            self.filtered_after = []

        def step(self):
            self.initialise()
            self.one_timestep(self.dt)
            if self.freq and self.tool_count % self.freq == 0:
                for pa in self.o.pas:
                    if pa.name in self.names:
                        density_filter(pa, self.corr, self.filter_kernel, self.dim)
                self.filtered_after.append(self.count + 1)
            self.tool_count += 1
            self.t += self.dt
            self.count += 1
            self.dt = self._get_timestep()
    return Solver
