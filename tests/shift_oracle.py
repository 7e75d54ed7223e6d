"""TEST INFRASTRUCTURE: ShiftPositions' equations in fp64 numpy, and the oracle solvers with the
tool.

``shift`` restates SimpleShift / FickianShift (pysph/sph/wc/shift.py:41-148) and
``correct_velocities`` CorrectVelocities (:151-188), vectorised over the destinations, as the
device runs them: every dpos from the positions before the shift (a Jacobi update), sources the
array's own particles with the accept test of linked_list_nnps.pyx:188, periodic images the
nearest ones (the box is wider than twice the support); the kernel values come from the fp64
oracle (oracle.kernel_w, oracle.kernel_grad).  Each also returns N_NBRS and, per particle, the
sum of the absolute values of its terms (the scale the device's fp32 kernel values are judged
against).  ``with_shift`` adds the tool's post_step to an oracle solver class.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle import oracle as orc


def _pairs(pos, h, k, L):
    """(i, j, x_ij) with r^2 < (k h_i)^2 or r^2 < (k h_j)^2, sorted by i then j, the particle
    itself included; L[d] > 0: axis d is periodic with that period (nearest image)"""
    L = np.asarray(L, dtype=float)
    per = L > 0
    q = pos - pos.min(axis=0)
    q[:, per] = np.mod(pos[:, per], L[per])
    q[q >= np.where(per, L, np.inf)] = 0.0
    box = np.where(per, L, 4.0 * (np.ptp(pos, axis=0) + 1.0))
    tree = cKDTree(q, boxsize=box)
    pr = tree.query_pairs(k * float(np.max(h)) * (1 + 1e-9), output_type='ndarray')
    n = len(pos)
    i = np.concatenate([pr[:, 0], pr[:, 1], np.arange(n)])
    j = np.concatenate([pr[:, 1], pr[:, 0], np.arange(n)])
    d = pos[i] - pos[j]
    d[:, per] -= L[per] * np.round(d[:, per] / L[per])
    r2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
    ok = (r2 < (k * h[i]) ** 2) | (r2 < (k * h[j]) ** 2)
    o = np.lexsort((j[ok], i[ok]))
    return i[ok][o], j[ok][o], d[ok][o]


def gmax(kernel, dim, h):
    """the largest |grad W| of the kernel with smoothing length h: the scale of the fp32 kernel
    polynomial's rounding, which is absolute, not relative to the value (its pieces cancel)"""
    q = np.linspace(0.0, 3.0, 601)
    g1 = max(abs(orc.kernel_grad(kernel, dim, [r, 0.0, 0.0], r, 1.0)[0]) for r in q)
    return g1 * np.asarray(h, dtype=float) ** -(dim + 1)


def _grad(kernel, dim, xij, rij, hij):
    return np.array([orc.kernel_grad(kernel, dim, x, r, hh) for x, r, hh in zip(xij, rij, hij)]).reshape(-1, 3)


def shift(pos, vel, h, m, rho, kind, const, dt, kernel, dim, L=(0, 0, 0), tensile=False,
          tensile_const=0.2, tensile_pow=4, hdx=1.0):
    """dpos[n, 3], N_NBRS[n] and the per-particle scale: |fac| sum_j |term_ij| (simple), or
    |fac| sum_j |V_j (1 + f_ij)| max|grad W(h_ij)| (fickian)"""
    k = orc.load().orc_kernel_radius_scale(orc.K_IDS[kernel])
    n = len(pos)
    i, j, xij = _pairs(pos, h, k, L)
    rij = np.sqrt(np.sum(xij * xij, axis=1))
    nn = np.bincount(i, minlength=n)
    term = np.zeros((len(i), 3))
    if kind == 'simple':
        vmax = float(np.max(np.sqrt(vel[:, 0] ** 2 + vel[:, 1] ** 2 + vel[:, 2] ** 2)))
        term = xij / (rij ** 3 + 1e-08)[:, None]
        ri = np.bincount(i, weights=rij, minlength=n) / nn
        fac = const * ri * ri * vmax * dt
    else:
        hij = (h[i] + h[j]) * 0.5
        dw = _grad(kernel, dim, xij, rij, hij)
        f = m[j] / rho[j]
        if tensile:
            wij = np.array([orc.kernel_w(kernel, dim, r, hh) for r, hh in zip(rij, hij)])
            wdx = np.array([orc.kernel_w(kernel, dim, hh / hdx, hh) for hh in h])
            f = f * (1 + tensile_const * (wij / wdx[i]) ** tensile_pow)
        term = f[:, None] * dw
        fac = -const * h * np.sqrt(np.sum(vel * vel, axis=1)) * dt
        absterm = np.abs(f) * gmax(kernel, dim, hij)
    s = np.zeros((n, 3))
    a = np.zeros(n)
    for d in range(3):
        s[:, d] = np.bincount(i, weights=term[:, d], minlength=n)
    if kind == 'simple':
        absterm = np.sqrt(np.sum(term * term, axis=1))
    a = np.bincount(i, weights=absterm, minlength=n)
    return fac[:, None] * s, nn, np.abs(fac) * a


def correct_velocities(pos, vel, h, m, rho, dpos, kernel, dim, L=(0, 0, 0)):
    """the change of (u, v, w) [n, 3], N_NBRS[n] and the per-particle scale
    sum_j |V_j| |v_ij| max|grad W(h_ij)| |dpos_i|"""
    k = orc.load().orc_kernel_radius_scale(orc.K_IDS[kernel])
    n = len(pos)
    i, j, xij = _pairs(pos, h, k, L)
    rij = np.sqrt(np.sum(xij * xij, axis=1))
    dw = _grad(kernel, dim, xij, rij, (h[i] + h[j]) * 0.5)
    vij = vel[i] - vel[j]
    vj = m[j] / rho[j]
    gradv = np.zeros((n, 3, 3))      # gradv[i][b][a] = -sum V_j v_ij[a] DW_ij[b]
    for b in range(3):
        for a in range(3):
            gradv[:, b, a] = np.bincount(i, weights=-vj * vij[:, a] * dw[:, b], minlength=n)
    du = np.einsum('nkl,nl->nk', gradv, dpos)
    hij = (h[i] + h[j]) * 0.5
    mag = np.bincount(i, weights=np.abs(vj) * np.linalg.norm(vij, axis=1) * gmax(kernel, dim, hij),
                      minlength=n)
    return du, np.bincount(i, minlength=n), mag * np.linalg.norm(dpos, axis=1)


def apply_tool(pa, kind, const, dt, kernel, dim, L, correct, wrap=None):
    """ShiftPositions' post_step on the real particles of ``pa`` (in place): shift; with the
    correction, ``wrap()`` (the domain update the device makes before it) and correct."""
    nr = pa.get_number_of_particles(real=True)
    P = pa.properties

    def state():
        pos = np.stack([P[c][:nr] for c in 'xyz'], axis=1)
        vel = np.stack([P[c][:nr] for c in 'uvw'], axis=1)
        return pos, vel, P['h'][:nr], P['m'][:nr], P['rho'][:nr]
    pos, vel, h, m, rho = state()
    dpos = shift(pos, vel, h, m, rho, kind, const, dt, kernel, dim, L)[0]
    for d, c in enumerate('xyz'):
        P[c][:nr] += dpos[:, d]
    if correct:
        if wrap is not None:
            pa = wrap()
            P = pa.properties
        pos, vel, h, m, rho = state()
        du = correct_velocities(pos, vel, h, m, rho, dpos, kernel, dim, L)[0]
        for d, c in enumerate('uvw'):
            P[c][:nr] += du[:, d]


def with_shift(base):
    """``base`` (an oracle solver class with a periodic or no domain) with ShiftPositions'
    post_step after every step, before t and dt advance (solver.py:480-491)."""

    class Solver(base):
        def __init__(self, particles, params, kernel, name='fluid', freq=1, kind='simple',
                     correct=False, const=None, dt=None, **kw):
            base.__init__(self, particles, params, kernel, **kw)
            self.name, self.freq, self.kind, self.correct = name, freq, kind, correct
            self.const = const or (0.04 if kind == 'simple' else 4)
            self.tool_dt = self.dt if dt is None else dt
            self.tool_count = 1
            self.shifted_after = []

        def _array(self):
            return [pa for pa in self.pas if pa.name == self.name][0]

        def _tool(self):
            dom = getattr(self, 'domain', None)
            L = [0.0, 0.0, 0.0]
            if dom is not None:
                L = [(dom[1][d] - dom[0][d]) if dom[2][d] else 0.0 for d in range(3)]

            def wrap():
                self.update_domain()
                return self._array()
            apply_tool(self._array(), self.kind, self.const, self.tool_dt, self.kernel, self.dim, L,
                       self.correct, wrap)
            self.update_domain()

        def _post_step(self, step):
            if self.freq and self.tool_count % self.freq == 0:
                self._tool()
                self.shifted_after.append(step)
            self.tool_count += 1

        def step(self):
            if hasattr(self, 'one_timestep'):        # WCSPH, TVD-RK3: adaptive dt
                self.initialise()
                self.one_timestep(self.dt)
                self._post_step(self.count + 1)
                self.t += self.dt
                self.count += 1
                self.dt = self._get_timestep()
            else:                                    # EDAC: fixed dt, t and count advance in step
                base.step(self)
                self._post_step(self.count)
    return Solver
