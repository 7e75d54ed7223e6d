"""TEST INFRASTRUCTURE: IISPHScheme's Groups (pysph/sph/iisph.py:37-402, :511-643) and
EulerIntegrator with IISPHStep (:22-34) in fp64 numpy, vectorised over the destinations.

Arrays are dicts name -> {'x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'p', ...} of fp64
numpy arrays; ``evaluate`` writes the scheme's properties into them as the reference does.
Neighbours are every (destination, source) pair with r^2 < (k h_i)^2 or r^2 < (k h_j)^2, the
particle itself included (linked_list_nnps.pyx:188); with a periodic box (L[d] > 0) the nearest
image, which is what the reference's ghost layer supplies when the box is wider than twice the
support.  The pressure iterations follow acceleration_eval_cython.mako:305-358: every
destination array's loop before its post-loop, the next array reading the pressures the last
one just solved, then PressureSolve.reduce of every fluid and the Group's iteration test.
"""
import numpy as np
from scipy.spatial import cKDTree

KERNELS = ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
RADIUS = {'CubicSpline': 2.0, 'WendlandQuintic': 2.0, 'QuinticSpline': 3.0, 'Gaussian': 3.0}


def _fac(kernel, dim):
    """the kernels' normalisation (pysph/base/kernels.py)"""
    if kernel == 'CubicSpline':
        return {1: 2.0 / 3.0, 2: 10.0 / np.pi / 7.0, 3: 1.0 / np.pi}[dim]
    if kernel == 'WendlandQuintic':
        return {2: 7.0 / np.pi / 4.0, 3: 21.0 / np.pi / 16.0}[dim]
    if kernel == 'QuinticSpline':
        return {1: 1.0 / 120.0, 2: 7.0 / np.pi / 478.0, 3: 1.0 / np.pi / 120.0}[dim]
    f = 1.0
    for _ in range(dim):
        f *= 0.5 * (2.0 / np.sqrt(np.pi))
    return f


def kernel_w_dwdq(kernel, dim, rij, h):
    """W(r, h) and dW/dq (times the normalisation, not yet / h) of kernels.py, vectorised"""
    h1 = 1.0 / h
    q = rij * h1
    fac = _fac(kernel, dim) * h1 ** dim
    w = np.zeros_like(q)
    dw = np.zeros_like(q)
    if kernel == 'CubicSpline':
        t2 = 2.0 - q
        a, b = q > 2.0, (q > 1.0) & (q <= 2.0)
        c = q <= 1.0
        w[b] = 0.25 * t2[b] ** 3
        w[c] = 1 - 1.5 * q[c] * q[c] * (1 - 0.5 * q[c])
        dw[b] = -0.75 * t2[b] * t2[b]
        dw[c] = -3.0 * q[c] * (1 - 0.75 * q[c])
        del a
    elif kernel == 'WendlandQuintic':
        t = 1.0 - 0.5 * q
        c = q < 2.0
        w[c] = t[c] ** 4 * (2.0 * q[c] + 1.0)
        dw[c] = -5.0 * q[c] * t[c] ** 3
    elif kernel == 'QuinticSpline':
        t3, t2, t1 = 3.0 - q, 2.0 - q, 1.0 - q
        a = (q > 2.0) & (q <= 3.0)
        b = (q > 1.0) & (q <= 2.0)
        c = q <= 1.0
        w[a] = t3[a] ** 5
        w[b] = t3[b] ** 5 - 6.0 * t2[b] ** 5
        w[c] = t3[c] ** 5 - 6.0 * t2[c] ** 5 + 15.0 * t1[c] ** 5
        dw[a] = -5.0 * t3[a] ** 4
        dw[b] = -5.0 * t3[b] ** 4 + 30.0 * t2[b] ** 4
        dw[c] = -5.0 * t3[c] ** 4 + 30.0 * t2[c] ** 4 - 75.0 * t1[c] ** 4
    else:
        c = q < 3.0
        w[c] = np.exp(-q[c] * q[c])
        dw[c] = -2.0 * q[c] * np.exp(-q[c] * q[c])
    dw[rij <= 1e-12] = 0.0
    return w * fac, dw * fac


def pairs(dst, src, kernel, L=(0.0, 0.0, 0.0), same=False):
    """(i, j, x_ij, r_ij, h_ij, W_ij, DW_ij) of the accepted (destination, source) pairs"""
    k = RADIUS[kernel]
    L = np.asarray(L, dtype=float)
    per = L > 0
    pd = np.stack([dst['x'], dst['y'], dst['z']], axis=1)
    ps = np.stack([src['x'], src['y'], src['z']], axis=1)
    if len(pd) == 0 or len(ps) == 0:
        e = np.zeros(0, dtype=np.int64)
        return e, e, np.zeros((0, 3)), np.zeros(0), np.zeros(0)
    lo = np.minimum(pd.min(axis=0), ps.min(axis=0))
    span = np.maximum(pd.max(axis=0), ps.max(axis=0)) - lo
    box = np.where(per, L, 4.0 * (span + 1.0))

    def fold(p):
        q = p - lo
        q[:, per] = np.mod(q[:, per], L[per])
        q[q >= box] = 0.0
        return q
    hmax = max(float(np.max(dst['h'])), float(np.max(src['h'])))
    td, ts = cKDTree(fold(pd), boxsize=box), cKDTree(fold(ps), boxsize=box)
    lst = td.query_ball_tree(ts, k * hmax * (1 + 1e-9))
    i = np.repeat(np.arange(len(pd)), [len(x) for x in lst]).astype(np.int64)
    j = np.array([y for x in lst for y in x], dtype=np.int64)
    d = pd[i] - ps[j]
    d[:, per] -= L[per] * np.round(d[:, per] / L[per])
    r2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
    ok = (r2 < (k * dst['h'][i]) ** 2) | (r2 < (k * src['h'][j]) ** 2)
    i, j, d, r2 = i[ok], j[ok], d[ok], r2[ok]
    r = np.sqrt(r2)
    hij = 0.5 * (dst['h'][i] + src['h'][j])
    return i, j, d, r, hij


def _kern(kernel, dim, pr):
    i, j, d, r, hij = pr
    w, dwdq = kernel_w_dwdq(kernel, dim, r, hij)
    tmp = np.where(r > 1e-12, dwdq / hij / np.where(r > 1e-12, r, 1.0), 0.0)
    return w, tmp[:, None] * d


def _sum(i, n, vals):
    if vals.ndim == 1:
        return np.bincount(i, weights=vals, minlength=n)
    return np.stack([np.bincount(i, weights=vals[:, c], minlength=n) for c in range(vals.shape[1])], axis=1)


def evaluate(arrays, fluids, solids, rho0, kernel, dim, dt, nu=0.0, g=(0.0, 0.0, 0.0), omega=0.5,
             tolerance=1e-2, min_iterations=2, max_iterations=30, L=(0.0, 0.0, 0.0)):
    """IISPHScheme.get_equations() once; writes V (solids), rho, uadv.., dii, rho_adv, aii, p0,
    piter, dijpj, p, compression, au.., dt_cfl, dt_force.  Returns (iterations, the list of
    {fluid: compression} after each iteration)."""
    PR, KW = {}, {}

    def nb(d, s):
        if (d, s) not in PR:
            PR[d, s] = pairs(arrays[d], arrays[s], kernel, L)
            KW[d, s] = _kern(kernel, dim, PR[d, s])
        return PR[d, s], KW[d, s]
    for s in solids:                                   # NumberDensity (:37-42)
        (i, j, *_), (w, dw) = nb(s, s)
        arrays[s]['V'] = _sum(i, len(arrays[s]['x']), w)
    for f in fluids:                                   # SummationDensity(+Boundary) (:45-59)
        A = arrays[f]
        n = len(A['x'])
        rho = np.zeros(n)
        for s in fluids:
            (i, j, *_), (w, dw) = nb(f, s)
            rho += _sum(i, n, arrays[s]['m'][j] * w)
        for s in solids:
            (i, j, *_), (w, dw) = nb(f, s)
            rho += _sum(i, n, rho0 / arrays[s]['V'][j] * w)
        A['rho'] = rho
    vel = lambda a, idx=slice(None): np.stack([a['u'][idx], a['v'][idx], a['w'][idx]], axis=1)  # noqa: E731
    adv = lambda a, idx=slice(None): np.stack([a['uadv'][idx], a['vadv'][idx], a['wadv'][idx]], axis=1)  # noqa: E731
    for f in fluids:                                   # Group 4 (:79-160)
        A = arrays[f]
        n = len(A['x'])
        rho_i = A['rho']
        acc = np.tile(np.asarray(g, dtype=float), (n, 1))
        dii = np.zeros((n, 3))
        for s in fluids + solids:
            (i, j, d, r, hij), (w, dw) = nb(f, s)
            S = arrays[s]
            if s in fluids:
                dii += _sum(i, n, (-S['m'][j] / rho_i[i] ** 2)[:, None] * dw)
            else:
                dii += _sum(i, n, (-1.0 / rho_i[i] ** 2 * rho0 / S['V'][j])[:, None] * dw)
            if nu > 0.0:
                vij = vel(A, i) - vel(S, j)
                dwx = np.sum(dw * d, axis=1)
                eps = 0.01 * hij * hij
                if s in fluids:
                    fac = 2.0 * nu * S['m'][j] / (0.5 * (rho_i[i] + S['rho'][j])) * dwx / (r * r + eps)
                else:
                    fac = 2.0 * nu * (rho0 / (S['V'][j] * rho_i[i])) * dwx / (r * r + eps)
                acc += _sum(i, n, fac[:, None] * vij)
        A['dii0'], A['dii1'], A['dii2'] = dii[:, 0].copy(), dii[:, 1].copy(), dii[:, 2].copy()
        ua = vel(A) + dt * acc
        A['uadv'], A['vadv'], A['wadv'] = ua[:, 0].copy(), ua[:, 1].copy(), ua[:, 2].copy()
    for f in fluids:                                   # Group 5 (:163-225)
        A = arrays[f]
        n = len(A['x'])
        dii_i = np.stack([A['dii0'], A['dii1'], A['dii2']], axis=1)
        rho_adv = A['rho'].copy()
        aii = np.zeros(n)
        for s in fluids + solids:
            (i, j, d, r, hij), (w, dw) = nb(f, s)
            S = arrays[s]
            fac = (A['m'] / A['rho'] ** 2)[i]
            dd = np.sum((dii_i[i] - fac[:, None] * dw) * dw, axis=1)
            if s in fluids:
                vd = np.sum((adv(A, i) - adv(S, j)) * dw, axis=1)
                rho_adv += _sum(i, n, dt * S['m'][j] * vd)
                aii += _sum(i, n, S['m'][j] * dd)
            else:
                phi = rho0 / S['V'][j]
                vd = np.sum((adv(A, i) - vel(S, j)) * dw, axis=1)
                rho_adv += _sum(i, n, dt * phi * vd)
                aii += _sum(i, n, phi * dd)
        A['rho_adv'], A['aii'] = rho_adv, aii
        A['p0'] = A['p'].copy()
        A['piter'] = 0.5 * A['p']
    history = []
    it = 1
    dt2 = dt * dt
    while True:                                        # Group(iterate=True) (:588-627)
        for f in fluids:                               # ComputeDIJPJ (:228-240)
            A = arrays[f]
            n = len(A['x'])
            dij = np.zeros((n, 3))
            for s in fluids:
                (i, j, *_), (w, dw) = nb(f, s)
                S = arrays[s]
                dij += _sum(i, n, (-S['m'][j] / S['rho'][j] ** 2 * S['piter'][j])[:, None] * dw)
            A['dijpj0'], A['dijpj1'], A['dijpj2'] = dij[:, 0].copy(), dij[:, 1].copy(), dij[:, 2].copy()
        comp = {}
        for f in fluids:                               # PressureSolve(+Boundary) (:264-355)
            A = arrays[f]
            n = len(A['x'])
            dpi = np.stack([A['dijpj0'], A['dijpj1'], A['dijpj2']], axis=1)
            acc = np.zeros(n)
            for s in fluids + solids:
                (i, j, *_), (w, dw) = nb(f, s)
                S = arrays[s]
                if s in fluids:
                    fac = (A['m'] / A['rho'] ** 2 * A['piter'])[i]
                    djk = np.stack([S['dijpj0'][j], S['dijpj1'][j], S['dijpj2'][j]], axis=1) - fac[:, None] * dw
                    sdii = np.stack([S['dii0'][j], S['dii1'][j], S['dii2'][j]], axis=1)
                    tmp = dpi[i] - sdii * S['piter'][j][:, None] - djk
                    acc += _sum(i, n, S['m'][j] * np.sum(tmp * dw, axis=1))
                else:
                    acc += _sum(i, n, rho0 / S['V'][j] * np.sum(dpi[i] * dw, axis=1))
            tmp = rho0 - A['rho_adv'] - acc * dt2
            dnr = A['aii'] * dt2
            big = np.abs(dnr) > 1e-9
            p = np.zeros(n)
            p[big] = np.maximum((1.0 - omega) * A['piter'][big] + omega / dnr[big] * tmp[big], 0.0)
            A['compression'] = np.where(p != 0.0, np.abs(p * dnr - tmp) + rho0, rho0)
            A['piter'] = p.copy()
            A['p'] = p.copy()
            c = A['compression']
            cnt, tot = float(np.sum(c > 0.0)), float(np.sum(c))
            avg = tot / cnt if cnt > 0 else rho0
            comp[f] = abs(avg - rho0) / rho0
        history.append(comp)
        conv = all(not (c > tolerance) for c in comp.values())
        if it >= min_iterations and (conv or it == max_iterations):
            break
        it += 1
    for f in fluids:                                   # PressureForce(+Boundary) (:367-402)
        A = arrays[f]
        n = len(A['x'])
        acc = np.zeros((n, 3))
        pi = A['p'] / A['rho'] ** 2
        for s in fluids + solids:
            (i, j, *_), (w, dw) = nb(f, s)
            S = arrays[s]
            if s in fluids:
                fac = -S['m'][j] * (pi[i] + S['p'][j] / S['rho'][j] ** 2)
            else:
                fac = -pi[i] * rho0 / S['V'][j]
            acc += _sum(i, n, fac[:, None] * dw)
        A['au'], A['av'], A['aw'] = acc[:, 0].copy(), acc[:, 1].copy(), acc[:, 2].copy()
        A['dt_cfl'] = 2.0 * np.sqrt(A['uadv'] ** 2 + A['vadv'] ** 2 + A['wadv'] ** 2)
        A['dt_force'] = 2.0 * np.sum(acc * acc, axis=1)
    return it, history


def stage(A, dt, L=(0.0, 0.0, 0.0), lo=(0.0, 0.0, 0.0)):
    """IISPHStep.stage1 (:22-34), then the periodic wrap of update_domain"""
    for c, a in (('u', 'au'), ('v', 'av'), ('w', 'aw')):
        A[c] = A[c + 'adv'] + dt * A[a]
    for x, u in (('x', 'u'), ('y', 'v'), ('z', 'w')):
        A[x] = A[x] + dt * A[u]
    for d, x in enumerate('xyz'):
        if L[d] > 0:
            A[x] = lo[d] + np.mod(A[x] - lo[d], L[d])


def dt_factors(arrays, names):
    """Integrator._get_dt_adapt_factors / compute_h_minimum (integrator.py:62-81, :146-159)
    over the arrays that carry dt_cfl / dt_force"""
    have = [n for n in names if 'dt_cfl' in arrays[n] and arrays[n]['dt_cfl'].size]
    cfl = max([float(np.max(arrays[n]['dt_cfl'])) for n in have] or [-1.0])
    force = max([float(np.max(arrays[n]['dt_force'])) for n in have] or [-1.0])
    hmin = min([1.0] + [float(np.min(arrays[n]['h'])) for n in names if arrays[n]['h'].size])
    return cfl, force, hmin


class Solver(object):
    """EulerIntegrator + IISPHStep for every fluid (IISPHScheme.configure_solver, :469-509), with
    the reference Solver's fixed or adaptive dt (solver.py:647-688: dt = cfl min(hmin / max
    dt_cfl, sqrt(hmin / sqrt(max dt_force))), no damping)."""

    def __init__(self, arrays, fluids, solids, rho0, kernel, dim, dt, L=(0.0, 0.0, 0.0),
                 lo=(0.0, 0.0, 0.0), adaptive=False, cfl=0.3, **kw):
        self.arrays, self.fluids, self.solids = arrays, list(fluids), list(solids)
        self.rho0, self.kernel, self.dim, self.dt = rho0, kernel, dim, dt
        self.L, self.lo, self.adaptive, self.cfl, self.kw = L, lo, adaptive, cfl, kw
        self.iterations, self.history = [], []
        self.t = 0.0
        self.fixed_hmin = None

    def evaluate(self, dt):
        it, hist = evaluate(self.arrays, self.fluids, self.solids, self.rho0, self.kernel, self.dim, dt,
                            L=self.L, **self.kw)
        self.iterations.append(it)
        self.history.append(hist)

    def margin(self):
        """the smallest |log(compression / tolerance)| at an iteration where the Group's test
        was made (it >= min_iterations): how far every decision was from the tolerance"""
        tol = self.kw.get('tolerance', 1e-2)
        m = np.inf
        for hist in self.history:
            for k, h in enumerate(hist):
                if k + 1 >= self.kw.get('min_iterations', 2):
                    m = min([m] + [abs(np.log(c / tol)) for c in h.values() if c > 0])
        return m

    def next_dt(self):
        if not self.adaptive:
            return self.dt
        f_cfl, f_force, hmin = dt_factors(self.arrays, list(self.arrays))
        if self.fixed_hmin is None:
            self.fixed_hmin = hmin
        hmin = self.fixed_hmin
        c = hmin / f_cfl if f_cfl > 0 else np.inf
        f = np.sqrt(hmin / np.sqrt(f_force)) if f_force > 0 else np.inf
        m = min(c, f)
        return self.dt if (m <= 0.0 or np.isinf(m)) else self.cfl * m

    def initialise(self):
        self.evaluate(self.dt)                        # solver.py:454 initial_acceleration
        self.dt = self.next_dt()

    def step(self):
        self.evaluate(self.dt)
        for f in self.fluids:
            stage(self.arrays[f], self.dt, self.L, self.lo)
        self.t += self.dt
        self.dt = self.next_dt()
