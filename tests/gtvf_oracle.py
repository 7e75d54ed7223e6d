"""TEST INFRASTRUCTURE: GTVFScheme's two evaluations (pysph/sph/wc/gtvf.py:586-662, with
transport_velocity.py's wall equations) and GTVFIntegrator with GTVFStep (:52-98) in fp64 numpy,
vectorised over the destinations.

Arrays are dicts name -> {'x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'p', 'uhat', ...} of
fp64 numpy arrays; ``evaluate0`` / ``evaluate1`` write the scheme's properties into them as the
reference does.  Neighbours are iisph_oracle.pairs': every (destination, source) pair with
r^2 < (k h_i)^2 or r^2 < (k h_j)^2, the particle itself included, with the nearest image in a
periodic box.  One fluid array (the device refuses more).
"""
import numpy as np

from iisph_oracle import KERNELS, RADIUS, kernel_w_dwdq, pairs, _sum  # noqa: F401


def _grad(kernel, dim, pr, scale=1.0):
    """W and grad W at scale * h_ij of the pairs pr"""
    i, j, d, r, hij = pr
    h = scale * hij
    w, dwdq = kernel_w_dwdq(kernel, dim, r, h)
    tmp = np.where(r > 1e-12, dwdq / h / np.where(r > 1e-12, r, 1.0), 0.0)
    return w, tmp[:, None] * d


def _vec(A, names, idx=slice(None)):
    return np.stack([A[n][idx] for n in names], axis=1)


class _Pairs(object):
    def __init__(self, arrays, kernel, dim, L):
        self.arrays, self.kernel, self.dim, self.L = arrays, kernel, dim, L
        self.cache = {}

    def __call__(self, d, s):
        if (d, s) not in self.cache:
            pr = pairs(self.arrays[d], self.arrays[s], self.kernel, self.L)
            self.cache[d, s] = pr, _grad(self.kernel, self.dim, pr)
        return self.cache[d, s]


def evaluate0(arrays, fluids, solids, kernel, dim, L=(0.0, 0.0, 0.0)):
    """SetWallVelocity of every wall, then ContinuityEquationGTVF + ContinuitySolid"""
    nb = _Pairs(arrays, kernel, dim, L)
    for s in solids:                                   # tv:100-134
        W = arrays[s]
        n = len(W['x'])
        wij, uf = np.zeros(n), np.zeros((n, 3))
        for f in fluids:
            (i, j, *_), (w, dw) = nb(s, f)
            wij += _sum(i, n, w)
            uf += _sum(i, n, w[:, None] * _vec(arrays[f], 'uvw', j))
        big = wij > 1e-12
        uf[big] /= wij[big][:, None]
        W['wij'] = wij
        for c, k in enumerate('uvw'):
            W[k + 'f'] = uf[:, c].copy()
            W[k + 'g'] = 2.0 * W[k] - uf[:, c]
    for f in fluids:                                   # gtvf.py:110-121, tv:164-173
        A = arrays[f]
        n = len(A['x'])
        arho = np.zeros(n)
        for s in fluids + solids:
            (i, j, *_), (w, dw) = nb(f, s)
            S = arrays[s]
            if s in fluids:
                vij = _vec(A, ('uhat', 'vhat', 'what'), i) - _vec(S, ('uhat', 'vhat', 'what'), j)
            else:
                vij = _vec(A, 'uvw', i) - _vec(S, ('ug', 'vg', 'wg'), j)
            arho += _sum(i, n, A['rho'][i] * S['m'][j] / S['rho'][j] * np.sum(dw * vij, axis=1))
        A['arho'] = arho


def evaluate1(arrays, fluids, solids, kernel, dim, rho0, pref, c0=0.0, alpha=0.0, nu=0.0,
              g=(0.0, 0.0, 0.0), L=(0.0, 0.0, 0.0)):
    """CorrectDensity + StateEquation, VolumeSummation + SolidWallPressureBC, the momentum Group"""
    nb = _Pairs(arrays, kernel, dim, L)
    all_ = fluids + solids
    for f in fluids:                                   # gtvf.py:138-148
        arrays[f]['rho0'] = arrays[f]['rho'].copy()
    for f in fluids:
        A = arrays[f]
        n = len(A['x'])
        rho, div = np.zeros(n), np.zeros(n)
        for s in all_:
            (i, j, *_), (w, dw) = nb(f, s)
            S = arrays[s]
            mw = S['m'][j] * w
            rho += _sum(i, n, mw)
            with np.errstate(divide='ignore', invalid='ignore'):
                div += _sum(i, n, mw / S['rho0'][j])
        A['rhodiv'] = div
        A['rho'] = rho / np.where(div < 1.0, div, 1.0)
        A['p'] = pref * (A['rho'] / rho0 - 1.0)        # tv:215-216, b = 1
    g = np.asarray(g, dtype=float)
    for s in solids:                                   # tv:71-75, :711-736
        W = arrays[s]
        n = len(W['x'])
        V, p, wij = np.zeros(n), np.zeros(n), np.zeros(n)
        gw = g[None, :] - _vec(W, ('au', 'av', 'aw'))
        for src in all_:
            (i, j, d, r, hij), (w, dw) = nb(s, src)
            V += _sum(i, n, w)
            if src in fluids:
                S = arrays[src]
                gdx = np.sum(gw[i] * d, axis=1)
                p += _sum(i, n, S['p'][j] * w + S['rho'][j] * gdx * w)
                wij += _sum(i, n, w)
        big = wij > 1e-14
        p[big] /= wij[big]
        W['V'], W['p'], W['wij'] = V, p, wij
        W['rho'] = rho0 * (p / pref + 1.0)
    for f in fluids:                                   # the momentum Group
        A = arrays[f]
        n = len(A['x'])
        acc = np.zeros((n, 3)) if alpha > 0.0 else np.tile(g, (n, 1))
        acch = np.zeros((n, 3))
        p0 = np.minimum(10.0 * np.abs(A['p']), pref)
        rhoi = A['rho']
        ui = _vec(A, 'uvw')
        uhi = _vec(A, ('uhat', 'vhat', 'what'))
        for s in all_:
            (i, j, d, r, hij), (w, dw) = nb(f, s)
            S = arrays[s]
            rj, mj = S['rho'][j], S['m'][j]
            ri = rhoi[i]
            fp = -mj * (A['p'][i] / ri ** 2 + S['p'][j] / rj ** 2)      # gtvf.py:232-241
            acc += _sum(i, n, fp[:, None] * dw)
            _, dwh = _grad(kernel, dim, (i, j, d, r, hij), 0.5)          # gtvf.py:243-250
            acch += _sum(i, n, (-p0[i] * mj / ri ** 2)[:, None] * dwh)
            vij = ui[i] - _vec(S, 'uvw', j)
            eps = 0.01 * hij * hij
            r2 = r * r
            if alpha > 0.0:                                              # tv:432-448
                vr = np.sum(vij * d, axis=1)
                mu = hij * vr / (r2 + eps)
                pij = np.where(vr < 0.0, mj * (-alpha * c0 * mu) / (0.5 * (ri + rj)), 0.0)
                acc += _sum(i, n, -pij[:, None] * dw)
            if nu > 0.0:                                                 # gtvf.py:274-288
                etai, etaj = nu * ri, nu * rj
                etaij = 4.0 * (etai * etaj) / (etai + etaj)
                fac = mj / (ri * rj) * etaij * np.sum(dw * d, axis=1) / (r2 + eps)
                acc += _sum(i, n, fac[:, None] * vij)
            if s in fluids:                                              # gtvf.py:309-348
                uj = _vec(S, 'uvw', j)
                dj = _vec(S, ('uhat', 'vhat', 'what'), j) - uj
                di = uhi[i] - ui[i]
                Aij = ui[i][:, :, None] * di[:, None, :] / ri[:, None, None] + \
                    uj[:, :, None] * dj[:, None, :] / rj[:, None, None]
                res = np.einsum('kab,kb->ka', Aij, dw)
                acc += _sum(i, n, mj[:, None] * res)
        for c, k in enumerate('uvw'):
            A['a' + k] = acc[:, c].copy()
            A['a' + k + 'hat'] = acch[:, c].copy()
        A['p0'] = p0


def stage(A, which, dt, L=(0.0, 0.0, 0.0), lo=(0.0, 0.0, 0.0)):
    """GTVFStep.stage1 / 2 / 3 (gtvf.py:71-98); after stage 2 the periodic wrap of update_domain"""
    if which == 2:
        A['rho'] = A['rho'] + dt * A['arho']
        for x, u in (('x', 'uhat'), ('y', 'vhat'), ('z', 'what')):
            A[x] = A[x] + dt * A[u]
        for d, x in enumerate('xyz'):
            if L[d] > 0:
                A[x] = lo[d] + np.mod(A[x] - lo[d], L[d])
        return
    for k in 'uvw':
        A[k] = A[k] + 0.5 * dt * A['a' + k]
        if which == 1:
            A[k + 'hat'] = A[k] + 0.5 * dt * A['a' + k + 'hat']


class Solver(object):
    """GTVFIntegrator with GTVFStep for the fluid at a fixed dt: initial_acceleration runs
    evaluation 0, then every step stage1, evaluation 0, stage2, evaluation 1, stage3."""

    def __init__(self, arrays, fluids, solids, kernel, dim, dt, rho0, pref, L=(0.0, 0.0, 0.0),
                 lo=(0.0, 0.0, 0.0), **kw):
        self.arrays, self.fluids, self.solids = arrays, list(fluids), list(solids)
        self.kernel, self.dim, self.dt, self.rho0, self.pref = kernel, dim, dt, rho0, pref
        self.L, self.lo, self.kw = L, lo, kw
        self.t = 0.0

    def eval0(self):
        evaluate0(self.arrays, self.fluids, self.solids, self.kernel, self.dim, L=self.L)

    def eval1(self):
        evaluate1(self.arrays, self.fluids, self.solids, self.kernel, self.dim, self.rho0,
                  self.pref, L=self.L, **self.kw)

    def initialise(self):
        self.eval0()

    def step(self):
        for which in (1, 2, 3):
            for f in self.fluids:
                stage(self.arrays[f], which, self.dt, self.L, self.lo)
            if which == 1:
                self.eval0()
            elif which == 2:
                self.eval1()
        self.t += self.dt
