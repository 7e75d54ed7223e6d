"""Generate tests/golden/iisph_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's pysph/sph/iisph.py and
pysph/base/kernels.py are loaded by path, unmodified; IISPHScheme(...).get_equations() gives the
Groups, and a driver written after acceleration_eval_cython.mako:10-154 and :262-363 runs their
bodies:
  * per Group and destination (in order of first appearance): initialize over the destination's
    particles (the real ones for Group(real=True)), the no-source loops, then per source the
    loops over NBRS by brute force -- r^2 < (k h_i)^2 or r^2 < (k h_j)^2
    (linked_list_nnps.pyx:188), ascending, the particle itself included -- then post_loop and
    reduce;
  * Group(iterate=True): the sub-groups in turn until min_iterations are done and every
    equation's converged() > 0 or max_iterations are reached
    (acceleration_eval_cython_helper.py:320-340);
  * DWIJ, WIJ, HIJ, EPS, RHOIJ1, VIJ, XIJ, R2IJ as oracle/gen_golden.py forms them;
  * a periodic case (IISPHScheme(has_ghosts=True)) materialises every image of the box as ghost
    particles (tag 2, orig_idx) after the real ones, so UpdateGhostProps / UpdateGhostPressure
    have something to copy.  The inputs carry piter = p / 2, which the images copy: the first
    ComputeDIJPJ reads the images' piter before UpdateGhostProps refreshes it.  The box exceeds twice the support: a ghost that neighbours a real
    particle has its whole neighbourhood.  The ghosts enter PressureSolve.reduce with
    compression 0 (not counted);
  * then IISPHStep.stage1 (:22-34) on every real fluid particle with the evaluation's dt.
compyle's `declare` is stubbed to 0, serial_reduce_array to numpy and parallel_reduce_array to
the identity; Equation, Group, Scheme and IntegratorStep to plain bases.

    python tests/gen_iisph_golden.py
"""
import itertools
import json
import math
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden import REF, GOLD, _load, call, pair_symbols  # noqa: E402

KERNELS = ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
NAME = os.path.join(GOLD, 'iisph_cases.json')
OUT_FLUID = ('rho', 'rho_adv', 'dii0', 'dii1', 'dii2', 'aii', 'p', 'au', 'av', 'aw', 'uadv', 'vadv',
             'wadv', 'dt_cfl', 'dt_force')
PROPS = ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'p', 'V', 'au', 'av', 'aw', 'uadv', 'vadv',
         'wadv', 'rho_adv', 'dii0', 'dii1', 'dii2', 'aii', 'dijpj0', 'dijpj1', 'dijpj2', 'p0',
         'piter', 'compression', 'dt_cfl', 'dt_force', 'ax', 'ay', 'az', 'tag', 'orig_idx')


def load():
    for pkg in ('pysph', 'pysph.sph', 'pysph.base', 'compyle'):
        sys.modules.setdefault(pkg, types.ModuleType(pkg))
    api = types.ModuleType('compyle.api')
    api.declare = lambda kind, n=1: 0
    sys.modules['compyle.api'] = api
    pa = types.ModuleType('pysph.base.particle_array')
    pa.get_ghost_tag = lambda: 2
    sys.modules['pysph.base.particle_array'] = pa
    eq = types.ModuleType('pysph.sph.equation')

    class Equation(object):
        def __init__(self, dest, sources):
            self.dest = dest
            self.sources = sources

        def converged(self):          # equation.py:424-427
            return 1.0

    class Group(object):
        def __init__(self, equations, real=True, iterate=False, max_iterations=1,
                     min_iterations=0, **kw):
            self.equations = equations
            self.real = real
            self.iterate = iterate
            self.max_iterations = max_iterations
            self.min_iterations = min_iterations
            self.has_subgroups = len(equations) > 0 and isinstance(equations[0], Group)
    eq.Equation, eq.Group = Equation, Group
    sys.modules['pysph.sph.equation'] = eq
    st = types.ModuleType('pysph.sph.integrator_step')
    st.IntegratorStep = type('IntegratorStep', (object,), {})
    sys.modules['pysph.sph.integrator_step'] = st
    ra = types.ModuleType('pysph.base.reduce_array')
    ra.serial_reduce_array = lambda a, op: getattr(np, op)(a)
    ra.parallel_reduce_array = lambda a, op: a
    sys.modules['pysph.base.reduce_array'] = ra
    sc = types.ModuleType('pysph.sph.scheme')
    sc.Scheme = type('Scheme', (object,), {})
    sc.add_bool_argument = None
    sys.modules['pysph.sph.scheme'] = sc
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    iisph = _load('pysph.sph.iisph', os.path.join(REF, 'pysph/sph/iisph.py'))
    return kernels, iisph


def nbrs(d, s, i, k):
    """brute-force NBRS of destination i of d among every particle of s, ascending"""
    dx = [np.array(s[c]) - d[c][i] for c in 'xyz']
    r2 = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]
    hi, hj = k * d['h'][i], k * np.array(s['h'])
    return [int(j) for j in np.nonzero((r2 < hi * hi) | (r2 < hj * hj))[0]]


def do_group(g, arrays, kernel, nreal, dt, comp):
    k = kernel.radius_scale
    dests = []
    for e in g.equations:
        if e.dest not in dests:
            dests.append(e.dest)
    for dn in dests:
        d = arrays[dn]
        npd = nreal[dn] if g.real else len(d['x'])
        deqs = [e for e in g.equations if e.dest == dn]
        denv = dict(('d_' + p, v) for p, v in d.items())
        denv['dt'] = dt
        for i in range(npd):
            for e in deqs:
                if hasattr(e, 'initialize'):
                    call(e.initialize, dict(denv, d_idx=i))
        srcs = []
        for e in deqs:
            for s in (e.sources or []):
                if s not in srcs:
                    srcs.append(s)
        for sn in srcs:
            s = arrays[sn]
            seqs = [e for e in deqs if e.sources and sn in e.sources and hasattr(e, 'loop')]
            senv = dict(('s_' + p, v) for p, v in s.items())
            for i in range(npd):
                for j in nbrs(d, s, i, k):
                    env = dict(denv, **senv)
                    env.update(pair_symbols(kernel, d, s, i, j))
                    env.update(d_idx=i, s_idx=j)
                    for e in seqs:
                        call(e.loop, env)
        for i in range(npd):
            for e in deqs:
                if hasattr(e, 'post_loop'):
                    call(e.post_loop, dict(denv, d_idx=i))
        for e in deqs:
            if hasattr(e, 'reduce'):
                dst = types.SimpleNamespace(compression=np.array(d['compression']),
                                            tmp_comp=np.zeros(2))
                e.reduce(dst, 0.0, dt)
                comp[dn] = float(e.compression)


def converged(g):
    if g.has_subgroups:
        return all([converged(s) for s in g.equations])
    return all([e.converged() > 0 for e in g.equations])


def evaluate(groups, arrays, kernel, nreal, dt):
    """the Groups once; returns the iteration count and each iteration's compression"""
    history, iterations = [], 0
    for g in groups:
        if not g.iterate:
            do_group(g, arrays, kernel, nreal, dt, {})
            continue
        it = 1
        while True:
            comp = {}
            for sg in g.equations:
                do_group(sg, arrays, kernel, nreal, dt, comp)
            history.append(comp)
            if it >= g.min_iterations and (converged(g) or it == g.max_iterations):
                break
            it += 1
        iterations = it
    return iterations, history


def _short(v):
    return [float('%.6g' % x) for x in v]


def lattice(dim, nx, dx, origin):
    axes = [np.arange(nx[d]) * dx + origin[d] for d in range(dim)]
    pts = np.stack([g.ravel() for g in np.meshgrid(*axes, indexing='ij')], axis=1)
    return np.concatenate([pts, np.zeros((len(pts), 3 - dim))], axis=1)


def make_array(pts, rs, dx, dim, hdx, vel, rho0=1000.0):
    n = len(pts)
    v = np.zeros((n, 3))
    v[:, :dim] = vel * rs.uniform(-1, 1, (n, dim))
    a = dict(x=pts[:, 0], y=pts[:, 1], z=pts[:, 2], u=v[:, 0], v=v[:, 1], w=v[:, 2],
             h=hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)),
             m=rho0 * dx ** dim * (1.0 + 0.02 * rs.uniform(-1, 1, n)),
             rho=np.full(n, rho0), p=rho0 * 10.0 * rs.uniform(0, 1, n))
    a = dict((p, _short(x)) for p, x in a.items())
    # what ComputeRhoAdvection.initialize sets on the real particles; the ghosts copy it, so that
    # ComputeDIJPJ, which runs before UpdateGhostProps, reads the same piter on an image as on
    # its particle (the device's periodic images are the particles themselves)
    a['piter'] = [0.5 * x for x in a['p']]
    return a


def make_case(kind, dim, seed, k, dx=0.1):
    """kind: 'block' (a fluid block alone, converging), 'tank' (a block on a wall layer), 'two'
    (two fluid blocks side by side on a wall), 'periodic' (a jittered periodic box).  h varies
    by +-10 %.  No pair lies within 1e-9 (relative) of the accept radius.  Returns (arrays,
    fluids, solids, L)."""
    rs = np.random.RandomState(seed)
    nfl = {2: (5, 4), 3: (3, 3, 3)}[dim]
    L = 0.0
    if kind == 'periodic':
        nfl = {2: (8, 8), 3: (5, 5, 5)}[dim]
        hdx = 0.7 if k == 2 else 0.5
        L = nfl[0] * dx
        pts = lattice(dim, nfl, dx, [0.5 * dx] * 3)
        pts[:, :dim] += rs.uniform(-0.1, 0.1, (len(pts), dim)) * dx
        return dict(fluid=make_array(pts, rs, dx, dim, hdx, 1.0)), ['fluid'], [], L
    hdx = 1.2 if k == 2 else 0.8
    pts = lattice(dim, nfl, dx, [0.0] * 3)
    pts[:, :dim] += rs.uniform(-0.1, 0.1, (len(pts), dim)) * dx
    arrays = {}
    if kind == 'two':
        half = pts[:, 0] < 0.5 * (nfl[0] - 1) * dx
        arrays['fluid'] = make_array(pts[half], rs, dx, dim, hdx, 0.5)
        arrays['fluid2'] = make_array(pts[~half], rs, dx, dim, hdx, 0.5)
        fluids = ['fluid', 'fluid2']
    else:
        arrays['fluid'] = make_array(pts, rs, dx, dim, hdx, 1.0)
        fluids = ['fluid']
    solids = []
    if kind in ('tank', 'two'):
        wn = (nfl[0] + 2,) + ((nfl[1] + 2,) if dim == 3 else ()) + (2,)
        wall = lattice(dim, wn[:dim], dx, [-dx, -2.0 * dx, 0.0] if dim == 2 else [-dx, -dx, -2.0 * dx])
        w = make_array(wall, rs, dx, dim, hdx, 0.0)
        w['u'] = [0.1] * len(w['x'])        # a moving wall: s_u enters ComputeRhoBoundary
        arrays['wall'] = w
        solids = ['wall']
    return arrays, fluids, solids, L


def ghosts(arrays, dim, L):
    """every image of every particle (tag 2, orig_idx), after the real ones"""
    nreal = {}
    for name, a in arrays.items():
        n = len(a['x'])
        nreal[name] = n
        a['tag'] = [0] * n
        a['orig_idx'] = list(range(n))
        if not L:
            continue
        base = dict((p, list(v)) for p, v in a.items())
        for s in itertools.product((-1, 0, 1), repeat=dim):
            if not any(s):
                continue
            for p in base:
                if p in 'xyz' and 'xyz'.index(p) < dim and s['xyz'.index(p)]:
                    a[p] += [x + s['xyz'.index(p)] * L for x in base[p][:n]]
                elif p == 'tag':
                    a[p] += [2] * n
                else:
                    a[p] += list(base[p][:n])
    return nreal


def run_case(kernels, iisph, kname, dim, kind, seed, nu=0.0, tolerance=1e-2, g=(0.0, 0.0, 0.0),
             dt=2e-3):
    kernel = getattr(kernels, kname)(dim=dim)
    k = kernel.radius_scale
    while True:
        inputs, fluids, solids, L = make_case(kind, dim, seed, k)
        ok = True
        allp = [(np.stack([a[c] for c in 'xyz'], axis=1), np.array(a['h'])) for a in inputs.values()]
        for pa, ha in allp:
            for pb, hb in allp:
                for i in range(len(pa)):
                    dd = pb - pa[i]
                    if L:
                        dd[:, :dim] -= L * np.round(dd[:, :dim] / L)
                    r = np.sqrt(np.sum(dd * dd, axis=1))
                    for lim in (k * ha[i], k * hb):
                        if np.any(np.abs(r - lim) <= 1e-9 * lim):
                            ok = False
        if ok:
            break
        seed += 1000
    arrays = json.loads(json.dumps(inputs))
    for a in arrays.values():
        n = len(a['x'])
        for p in PROPS:
            a.setdefault(p, [0.0] * n)
    nreal = ghosts(arrays, dim, L)
    sch = iisph.IISPHScheme(fluids, solids, dim, 1000.0, nu=nu, gx=g[0], gy=g[1], gz=g[2],
                            tolerance=tolerance, has_ghosts=bool(L))
    it, hist = evaluate(sch.get_equations(), arrays, kernel, nreal, dt)
    out = dict(kernel=kname, dim=dim, kind=kind, seed=seed, nu=nu, tolerance=tolerance, g=list(g),
               dt=dt, L=L, fluids=fluids, solids=solids, inputs=inputs, iterations=it,
               compression=hist, rho0=1000.0, omega=0.5)
    res = {}
    for f in fluids:
        res[f] = dict((p, arrays[f][p][:nreal[f]]) for p in OUT_FLUID)
    for s in solids:
        res[s] = dict(V=arrays[s]['V'][:nreal[s]])
    step = iisph.IISPHStep()
    for f in fluids:
        a = arrays[f]
        for i in range(nreal[f]):
            call(step.stage1, dict([('d_' + p, v) for p, v in a.items()] + [('d_idx', i), ('dt', dt)]))
        res[f].update(dict(('step_' + p, a[p][:nreal[f]]) for p in 'xyzuvw'))
    out['outputs'] = res
    return out


# (kernel, dim) -> (geometry, nu, tolerance): every geometry, nu = 0 and nu > 0 beside walls,
# one case that stops at min_iterations (tolerance 1) and one that reaches max_iterations
PLAN = {
    ('CubicSpline', 2): ('tank', 0.0, 1e-2),
    ('CubicSpline', 3): ('block', 0.0, 1e-2),
    ('WendlandQuintic', 2): ('tank', 0.05, 1e-3),
    ('WendlandQuintic', 3): ('two', 0.0, 1e-2),
    ('QuinticSpline', 2): ('periodic', 0.01, 1e-3),
    ('QuinticSpline', 3): ('tank', 0.05, 1e-12),
    ('Gaussian', 2): ('two', 0.02, 1.0),
    ('Gaussian', 3): ('periodic', 0.0, 1e-2),
}


def gen_cases(kernels, iisph):
    cases = []
    seed = 700
    for kname in KERNELS:
        for dim in (2, 3):
            seed += 1
            kind, nu, tol = PLAN[kname, dim]
            g = (0.0, 0.0, 0.0) if kind in ('block', 'periodic') else \
                ((0.0, -9.81, 0.0) if dim == 2 else (0.0, 0.0, -9.81))
            cases.append(run_case(kernels, iisph, kname, dim, kind, seed, nu=nu, tolerance=tol, g=g))
            print(kname, dim, kind, 'iterations', cases[-1]['iterations'], flush=True)
    return cases


def main():
    kernels, iisph = load()
    iisph.sqrt, iisph.fabs = math.sqrt, math.fabs
    with open(NAME, 'w') as f:
        json.dump(gen_cases(kernels, iisph), f)
    print('wrote', NAME, os.path.getsize(NAME), 'bytes')


if __name__ == '__main__':
    main()
