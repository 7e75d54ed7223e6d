"""TEST INFRASTRUCTURE: the Interpolator's five methods (pysph/tools/interpolator.py:18-172) in
fp64 numpy over a golden case of tests/golden/interpolator_cases.json.

Sources are every particle of every array (images materialised in a periodic box, probes
wrapped into it, as tests/gen_interpolator_golden.py does); neighbours by the accept test
r^2 < (k h_d)^2 or r^2 < (k h_s)^2; W and its gradient from the fp64 oracle (oracle.kernel_w,
oracle.kernel_grad); gj_solve from tests/density_filter_oracle.py.  ``interpolate`` returns
what the Interpolator's ``pa.prop`` holds (4 values per probe for 'order1') and, for 'order1',
the condition number of each probe's moment matrix (inf where gj_solve returns early) and its
number of neighbours.
"""
import numpy as np

from oracle import oracle as orc
from density_filter_oracle import gj_solve

NAMES = ('fluid', 'solid')


def sources(case):
    cols = ('x', 'y', 'z', 'h', 'm', 'rho')
    src = dict((c, np.concatenate([np.array(case['arrays'][n][c]) for n in NAMES])) for c in cols)
    src['f'] = np.concatenate([np.array(case['arrays'][n].get('f', [0.0] * len(case['arrays'][n]['x'])))
                               for n in NAMES])
    box = case.get('box')
    if box is None:
        return src
    L = np.array(box['hi']) - np.array(box['lo'])
    shifts = [np.zeros(3)]
    for d in range(3):
        if box['periodic'][d]:
            shifts = [s + e * L[d] * np.eye(3)[d] for s in shifts for e in (-1, 0, 1)]
    out = dict((c, np.concatenate([src[c] + (s['xyz'.index(c)] if c in 'xyz' else 0.0) for s in shifts]))
               for c in src)
    return out


def probes(case):
    P = np.array([case['probes'][c] for c in 'xyz'], dtype=float)
    box = case.get('box')
    if box is not None:
        for d in range(3):
            if box['periodic'][d]:
                lo, hi = box['lo'][d], box['hi'][d]
                P[d] = np.where(P[d] < lo, P[d] + (hi - lo), P[d])
                P[d] = np.where(P[d] > hi, P[d] - (hi - lo), P[d])
    return P.T


def _pairs(q, hq, pos, h, k):
    """the sources j of each destination i, ascending"""
    out = []
    for i in range(len(q)):
        r2 = np.sum((pos - q[i]) ** 2, axis=1)
        out.append(np.nonzero((r2 < (k * hq[i]) ** 2) | (r2 < (k * h) ** 2))[0])
    return out


def interpolate(case, method, kernel=None, dim=None):
    kernel = kernel or case['kernel']
    dim = dim or case['dim']
    kid = orc.K_IDS[kernel]
    k = orc.load().orc_kernel_radius_scale(kid)
    src = sources(case)
    pos = np.stack([src['x'], src['y'], src['z']], axis=1)
    q = probes(case)
    npb = len(q)
    hp = max(max(case['arrays'][n]['h']) for n in NAMES)
    nb = _pairs(q, np.full(npb, hp), pos, src['h'], k)
    rho = src['rho']
    if method == 'order1':
        # Group(SummationDensity(dest=a, sources=all) for a), real=False
        rho = np.zeros(len(pos))
        for i, js in enumerate(_pairs(pos, src['h'], pos, src['h'], k)):
            for j in js:
                xij = pos[i] - pos[j]
                rho[i] += src['m'][j] * orc.kernel_w(kernel, dim, np.sqrt(xij @ xij), 0.5 * (src['h'][i] + src['h'][j]))
    V = src['m'] / rho
    res = np.zeros(npb * (4 if method == 'order1' else 1))
    cond = np.zeros(npb)
    for i, js in enumerate(nb):
        sw = sf = 0.0
        mom = np.zeros((4, 4))
        ps = np.zeros(4)
        for j in js:
            xij = q[i] - pos[j]
            rij = np.sqrt(xij @ xij)
            hs = src['h'][j]
            f = src['f'][j]
            if method == 'shepard':
                w = orc.kernel_w(kernel, dim, rij, 0.5 * (hp + hs))
                sw += w
                sf += w * f
            elif method == 'sph':
                sf += V[j] * orc.kernel_w(kernel, dim, rij, 0.5 * (hp + hs)) * f
            elif method == 'splash':
                sf += V[j] * orc.kernel_w(kernel, dim, rij, hp) * f
            elif method == 'splash_norm':
                c = V[j] * orc.kernel_w(kernel, dim, rij, hs)
                sw += c
                sf += c * f
            else:
                hij = 0.5 * (hp + hs)
                w = orc.kernel_w(kernel, dim, rij, hij)
                dw = np.array(orc.kernel_grad(kernel, dim, xij, rij, hij))
                mom[0, 0] += w * V[j]
                mom[0, 1:] += -xij * w * V[j]
                mom[1:, 0] += dw * V[j]
                mom[1:, 1:] += -np.outer(dw, xij) * V[j]
                ps[0] += f * w * V[j]
                ps[1:] += f * dw * V[j]
        if method == 'order1':
            n = dim + 1
            aug = np.zeros((1, n, n + 1))
            aug[0, :, :n] = mom[:n, :n]
            aug[0, :, n] = ps[:n]
            ok = gj_solve(aug)[0]
            if ok:
                res[4 * i:4 * i + n] = aug[0, :, n]
            with np.errstate(all='ignore'):
                cond[i] = np.linalg.cond(mom[:n, :n]) if ok else np.inf
        else:
            res[i] = sf / sw if method in ('shepard', 'splash_norm') and sw > 1e-12 else sf
    return (res, cond, np.array([len(js) for js in nb])) if method == 'order1' else res
