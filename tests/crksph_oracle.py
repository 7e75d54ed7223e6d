"""TEST INFRASTRUCTURE: CRKSPHScheme's two evaluations (pysph/sph/wc/crksph.py:978-1127) and
CRKSPHIntegrator with CRKSPHStep (:866-900) in fp64 numpy, vectorised over the pairs.

One fluid array: a dict of fp64 numpy arrays 'x', 'y', 'z', 'u', 'v', 'w', 'u0', 'v0', 'w0', 'h',
'm', 'rho', 'e'; ``evaluate0`` / ``evaluate1`` write p, cs, V, ai, bi (n, 3), gradai (n, 3),
gradbi (n, 3, 3) as [g][a], gradv (n, 3, 3) as [a][b], rho, au, av, aw and ae into it as the
reference does.  Neighbours are iisph_oracle.pairs': every (destination, source) pair with
r^2 < (k h_i)^2 or r^2 < (k h_j)^2, the particle itself included, with the nearest image in a
periodic box.  m2 is inverted by gj_solve's elimination without pivoting (linalg.py:94-166), with
its singular tests; min / max are Python's (the first argument unless the second compares below /
above it), so the limiter's 0 / 0 gives phi = 1.
"""
import numpy as np

from iisph_oracle import KERNELS, RADIUS, kernel_w_dwdq, pairs, _sum  # noqa: F401


def _wd(kernel, dim, x, r, h):
    w, dwdq = kernel_w_dwdq(kernel, dim, r, h)
    tmp = np.where(r > 1e-12, dwdq / h / np.where(r > 1e-12, r, 1.0), 0.0)
    return w, tmp[:, None] * x


def _pymin(a, b):
    return np.where(b < a, b, a)


def _pymax(a, b):
    return np.where(b > a, b, a)


def gj_inverse(M):
    """gj_solve on [M | I] for a batch (n, d, d): (inverse, singular)"""
    n, d, _ = M.shape
    m = np.concatenate([M, np.broadcast_to(np.eye(d), (n, d, d))], axis=2).copy()
    sing = np.zeros(n, dtype=bool)
    for c in range(d):
        for r in range(c + 1, d):
            piv = m[:, c, c].copy()
            bad = np.abs(piv) < 1e-12
            sing |= bad
            cc = -m[:, r, c] / np.where(bad, 1.0, piv)
            m[:, r, :] = np.where(sing[:, None], m[:, r, :], m[:, r, :] + cc[:, None] * m[:, c, :])
    for rb in range(d - 1, -1, -1):
        zero = m[:, rb, rb] == 0.0
        sing |= zero & (np.abs(m[:, rb, 2 * d - 1]) > 1e-12)
        ok = ~sing & ~zero
        piv = np.where(ok, m[:, rb, rb], 1.0)
        for bc in range(2 * d - 1, rb - 1, -1):
            m[:, rb, bc] = np.where(ok, m[:, rb, bc] / piv, m[:, rb, bc])
        for ku in range(rb - 1, -1, -1):
            kk = -m[:, ku, rb] / np.where(ok, m[:, rb, rb], 1.0)
            for kl in range(2 * d - 1, rb - 1, -1):
                m[:, ku, kl] = np.where(ok, m[:, ku, kl] + kk * m[:, rb, kl], m[:, ku, kl])
    return m[:, :, d:], sing


def _vec(A, names, idx=slice(None)):
    return np.stack([A[k][idx] for k in names], axis=1)


def _side(A, kernel, dim, k, sg, x, r):
    """one side of CRKSPHSymmetric (:354-388) for the particles k of the pairs"""
    wk, dwk = _wd(kernel, dim, x, r, A['h'][k])
    ak = A['ai'][k]
    bx = sg * np.einsum('pa,pa->p', A['bi'][k][:, :dim], x[:, :dim])
    dbx = sg * np.einsum('pga,pa->pg', A['gradbi'][k][:, :dim, :dim], x[:, :dim])
    t = ((sg * ak)[:, None] * dwk[:, :dim] + A['gradai'][k][:, :dim] * wk[:, None]) * (1 + bx)[:, None]
    t += ak[:, None] * (dbx + A['bi'][k][:, :dim]) * wk[:, None]
    return t


def _corrected(A, kernel, dim, pr):
    i, j, x, r, hij = pr
    _, dw = _wd(kernel, dim, x, r, hij)
    dwij = dw.copy()
    dwij[:, :dim] = 0.5 * (_side(A, kernel, dim, i, 1.0, x, r) - _side(A, kernel, dim, j, -1.0, x, r))
    return dwij


def _pq(A, dim, pr, vi, vj, cl, cq, eta_crit, eta_fold):
    i, j, x, r, hij = pr
    xd = x[:, :dim]
    G = A['gradv'][:, :dim, :dim]
    with np.errstate(divide='ignore', invalid='ignore'):
        tri = np.einsum('pab,pa,pb->p', G[i], xd, xd)
        trj = np.einsum('pab,pa,pb->p', G[j], xd, xd)
        rij = tri / trj
        tmprij = _pymin(1.0, 4 * rij / ((1 + rij) * (1 + rij)))
    phi = _pymax(0.0, tmprij)
    tx = np.sum(xd * xd, axis=1)
    tx2 = np.sqrt(tx)
    hi, hj = A['h'][i], A['h'][j]
    eta = _pymin(tx2 / hi, tx2 / hj)
    tmp = (eta - eta_crit) / eta_fold
    phi = np.where(eta < eta_crit, phi * np.exp(-tmp * tmp), phi)
    s = np.einsum('pab,pb->pa', G[i] + G[j], xd)
    uh = vi[:, :dim] - vj[:, :dim] - 0.5 * phi[:, None] * s
    ux = np.sum(uh * xd, axis=1)
    eps = 0.01 * hij * hij
    mui = _pymin(0.0, ux / (tx / hi + eps * hi))
    muj = _pymin(0.0, ux / (tx / hi + eps * hj))
    qi = A['rho'][i] * (-cl * A['cs'][i] * mui + cq * mui * mui)
    qj = A['rho'][j] * (-cl * A['cs'][j] * muj + cq * muj * muj)
    return A['p'][i] + A['p'][j] + qi + qj


def prestep(A, kernel, dim, pr):
    """CRKSPHPreStep.loop_all (:32-167): ai, bi, gradai, gradbi"""
    i, j, x, r, hij = pr
    n = len(A['x'])
    w, dw = _wd(kernel, dim, x, r, hij)
    Vj = 1.0 / A['V'][j]
    xd, dwd = x[:, :dim], dw[:, :dim]
    I = np.eye(dim)
    m0 = _sum(i, n, Vj * w)
    m1 = _sum(i, n, (Vj * w)[:, None] * xd)
    m2 = _sum(i, n, ((Vj * w)[:, None, None] * xd[:, :, None] * xd[:, None, :]).reshape(-1, dim * dim))
    m2 = m2.reshape(n, dim, dim)
    gm0 = _sum(i, n, Vj[:, None] * dwd)
    gm1 = Vj[:, None, None] * (dwd[:, :, None] * xd[:, None, :] + I[None] * w[:, None, None])   # [g][a]
    gm1 = _sum(i, n, gm1.reshape(-1, dim * dim)).reshape(n, dim, dim)
    t = xd[:, None, :, None] * I[None, :, None, :] + xd[:, None, None, :] * I[None, :, :, None]  # [g][a][b]
    gm2 = Vj[:, None, None, None] * (xd[:, None, :, None] * xd[:, None, None, :] * dwd[:, :, None, None]
                                     + t * w[:, None, None, None])
    gm2 = _sum(i, n, gm2.reshape(-1, dim ** 3)).reshape(n, dim, dim, dim)
    nn = np.bincount(i, minlength=n)
    inv, sing = gj_inverse(m2)
    tv = np.einsum('nab,nb->na', inv, m1)
    with np.errstate(divide='ignore', invalid='ignore'):
        ai = 1.0 / (m0 - np.sum(tv * m1, axis=1))
    bi = -tv
    t1 = gm0 - np.einsum('nab,nb,nga->ng', inv, m1, gm1) - np.einsum('nab,na,ngb->ng', inv, m1, gm1)
    K = np.einsum('nap,nqb,ngpq->ngab', inv, inv, gm2)
    t1 = t1 + np.einsum('ngab,nb,na->ng', K, m1, m1)
    gbi = -np.einsum('nab,ngb->nga', inv, gm1) + np.einsum('ngab,nb->nga', K, m1)
    gai = -ai[:, None] ** 2 * t1
    bad = sing | (nn < 2)
    A['ai'] = np.where(bad, 1.0, ai)
    A['bi'], A['gradai'], A['gradbi'] = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3, 3))
    A['bi'][:, :dim] = np.where(bad[:, None], 0.0, bi)
    A['gradai'][:, :dim] = np.where(bad[:, None], 0.0, gai)
    A['gradbi'][:, :dim, :dim] = np.where(bad[:, None, None], 0.0, gbi)


def _eos(A, gamma):
    A['p'] = (gamma - 1) * A['rho'] * A['e']
    with np.errstate(invalid='ignore'):
        A['cs'] = np.sqrt(gamma * A['p'] / A['rho'])


def evaluate0(A, kernel, dim, gamma=7.0, g=(0.0, 0.0, 0.0), cl=2, cq=1, eta_crit=0.3,
              eta_fold=0.2, nu=0.0, eta=0.01, L=(0.0, 0.0, 0.0)):
    """evaluation 0: StateEquation + SpeedOfSound, NumberDensity, CRKSPHPreStep, the CRKSPH
    density and StateEquation + SpeedOfSound, VelocityGradient, the momentum Group"""
    n = len(A['x'])
    pr = pairs(A, A, kernel, L)
    i, j, x, r, hij = pr
    _eos(A, gamma)
    w, _ = _wd(kernel, dim, x, r, A['h'][i])
    A['V'] = _sum(i, n, w)
    prestep(A, kernel, dim, pr)
    w, _ = _wd(kernel, dim, x, r, hij)
    Vj = 1.0 / A['V'][j]
    cw = A['ai'][i] * (1 + np.einsum('pa,pa->p', A['bi'][i], x))
    fac = Vj * cw * w
    A['rho'] = _sum(i, n, A['m'][i] * fac) / _sum(i, n, Vj * fac)
    _eos(A, gamma)
    dwi = _side(A, kernel, dim, i, 1.0, x, r)
    vij = _vec(A, 'uvw', i) - _vec(A, 'uvw', j)
    gv = -Vj[:, None, None] * vij[:, :dim, None] * dwi[:, None, :]
    A['gradv'] = np.zeros((n, 3, 3))
    A['gradv'][:, :dim, :dim] = _sum(i, n, gv.reshape(-1, dim * dim)).reshape(n, dim, dim)
    dwij = _corrected(A, kernel, dim, pr)
    pq = _pq(A, dim, pr, _vec(A, 'uvw', i), _vec(A, 'uvw', j), cl, cq, eta_crit, eta_fold)
    Vi = 1.0 / A['V'][i]
    f = -(1.0 / A['m'][i]) * Vi * Vj * pq
    acc = np.tile(np.asarray(g, dtype=float), (n, 1)) + _sum(i, n, f[:, None] * dwij)
    if abs(nu) > 1e-14:                                    # wc/viscosity.py:12-27
        fij = np.sum(dwij * x, axis=1)
        tmp = A['m'][j] * 4 * nu * fij / ((A['rho'][i] + A['rho'][j]) * (r * r + eta * hij * hij))
        acc += _sum(i, n, tmp[:, None] * vij)
    A['au'], A['av'], A['aw'] = acc[:, 0].copy(), acc[:, 1].copy(), acc[:, 2].copy()


def evaluate1(A, kernel, dim, gamma=7.0, cl=2, cq=1, eta_crit=0.5, eta_fold=0.2,
              L=(0.0, 0.0, 0.0)):
    """evaluation 1: CRKSPHSymmetric + EnergyEquation (its own defaults: eta_crit = 0.5)"""
    n = len(A['x'])
    pr = pairs(A, A, kernel, L)
    i, j, x, r, hij = pr
    dwij = _corrected(A, kernel, dim, pr)
    u0 = _vec(A, ('u0', 'v0', 'w0'))
    u = _vec(A, 'uvw')
    pq = _pq(A, dim, pr, u0[i], u0[j], cl, cq, eta_crit, eta_fold)
    Vi, Vj = 1.0 / A['V'][i], 1.0 / A['V'][j]
    f = -(1.0 / A['m'][i]) * Vi * Vj * pq
    delu = u0[j] + u[j] - u0[i] - u[i]
    aeij = np.sum(delu[:, :dim] * (f[:, None] * dwij[:, :dim]), axis=1)
    si = A['p'][i] / A['rho'][i] ** gamma
    sj = A['p'][j] / A['rho'][j] ** gamma
    smin, smax = _pymin(np.abs(si), np.abs(sj)), _pymax(np.abs(si), np.abs(sj))
    sd = si - sj
    with np.errstate(divide='ignore', invalid='ignore'):
        fij = np.where(sd * aeij > 0, smin / (smin + smax),
                       np.where(sd * aeij < 0, smax / (smin + smax), 0.5))
    A['ae'] = _sum(i, n, 0.5 * fij * aeij)


def stage(A, which, dt, L=(0.0, 0.0, 0.0), lo=(0.0, 0.0, 0.0)):
    """CRKSPHStep.stage1 / 2 / 3 (:885-900); after stage 3 the periodic wrap of update_domain"""
    if which == 1:
        for k in 'uvw':
            A[k + '0'] = A[k].copy()
    elif which == 2:
        for k in 'uvw':
            A[k] = A[k] + A['a' + k] * dt
    else:
        A['e'] = A['e'] + A['ae'] * dt
        for x, u in (('x', 'u'), ('y', 'v'), ('z', 'w')):
            A[x] = A[x] + 0.5 * dt * (A[u] + A[u + '0'])
        for d, x in enumerate('xyz'):
            if L[d] > 0:
                A[x] = lo[d] + np.mod(A[x] - lo[d], L[d])


class Solver(object):
    """CRKSPHIntegrator with CRKSPHStep at a fixed dt: initial_acceleration runs evaluation 0,
    then every step stage1, evaluation 0, stage2, evaluation 1, stage3."""

    def __init__(self, A, kernel, dim, dt, L=(0.0, 0.0, 0.0), lo=(0.0, 0.0, 0.0), **kw):
        self.A, self.kernel, self.dim, self.dt, self.L, self.lo = A, kernel, dim, dt, L, lo
        self.kw0 = dict((k, v) for k, v in kw.items() if k != 'gamma_e')
        self.gamma = kw.get('gamma', 7.0)
        self.t = 0.0

    def initialise(self):
        evaluate0(self.A, self.kernel, self.dim, L=self.L, **self.kw0)

    def step(self):
        stage(self.A, 1, self.dt)
        evaluate0(self.A, self.kernel, self.dim, L=self.L, **self.kw0)
        stage(self.A, 2, self.dt)
        evaluate1(self.A, self.kernel, self.dim, gamma=self.gamma, L=self.L)
        stage(self.A, 3, self.dt, self.L, self.lo)
        self.t += self.dt
