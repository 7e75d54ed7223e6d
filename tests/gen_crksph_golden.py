"""Generate tests/golden/crksph_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's pysph/sph/wc/crksph.py,
linalg.py, viscosity.py and pysph/base/kernels.py are loaded by path, unmodified;
CRKSPHScheme(...).get_equations() gives the two evaluations, and a driver written after
acceleration_eval_cython.mako:10-154 runs their bodies, with SPH_KERNEL the kernel object:
  * per Group and destination: initialize, the no-source loops, then per source the pair loops
    over NBRS by brute force -- r^2 < (k h_i)^2 or r^2 < (k h_j)^2 (linked_list_nnps.pyx:188),
    ascending, the particle itself included -- and loop_all with that NBRS and N_NBRS, then
    post_loop;
  * the pair symbols of oracle/gen_golden.py plus WI, WJ, DWI, DWJ (equation.py:245-283); the
    lists (DWIJ, DWI, DWJ) are shared by the equations of one pair, so CRKSPHSymmetric's
    corrections reach the equations after it, while its rebinding of WI / WJ does not;
  * a periodic case materialises every image of the box after the real particles (the box
    exceeds twice the support) and, after every Group, refreshes each image from its particle:
    the device's images are the particles themselves.  Only the real particles are destinations
    (an image's own results would be overwritten by the refresh);
  * properties are numpy fp64, so the limiter's r_ij = 0 / 0 of a vanishing gradv is nan and
    Python's min(1, nan) is 1.
compyle's `declare('matrix(n)')` is a list of n zeros and `declare('int')` a 0; Equation, Group,
MultiStageEquations, Scheme, Integrator and IntegratorStep are plain bases.

Each case records evaluation 0 and then evaluation 1 on the same inputs; cases with steps also
record that many CRKSPHIntegrator steps from the inputs (initial_acceleration, then stage1,
evaluation 0, stage2, evaluation 1, stage3).

    python tests/gen_crksph_golden.py
"""
import itertools
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden import REF, GOLD, _load, call, pair_symbols  # noqa: E402
from gen_iisph_golden import lattice, nbrs, _short  # noqa: E402

KERNELS = ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
NAME = os.path.join(GOLD, 'crksph_cases.json')
STRIDED = {'bi': 1, 'gradai': 1, 'gradbi': 2, 'gradv': 2}    # stride dim ** power
OUT0 = ('V', 'ai', 'bi', 'gradai', 'gradbi', 'rho', 'p', 'cs', 'gradv', 'au', 'av', 'aw')
OUT1 = ('ae',)
PROPS = ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'p', 'e', 'au', 'av', 'aw', 'ae', 'u0',
         'v0', 'w0', 'cs', 'V', 'rhofac', 'cwij', 'ai')


def declare(kind, n=1):
    if kind.startswith('matrix'):
        size = int(kind[kind.index('(') + 1:kind.index(')')])
        return [[0.0] * size for _ in range(n)] if n > 1 else [0.0] * size
    return tuple([0] * n) if n > 1 else 0


def load():
    for pkg in ('pysph', 'pysph.sph', 'pysph.sph.wc', 'pysph.base', 'compyle'):
        sys.modules.setdefault(pkg, types.ModuleType(pkg))
    api = types.ModuleType('compyle.api')
    api.declare = declare
    sys.modules['compyle.api'] = api
    pa = types.ModuleType('pysph.base.particle_array')
    pa.get_ghost_tag = lambda: 2
    sys.modules['pysph.base.particle_array'] = pa
    eq = types.ModuleType('pysph.sph.equation')

    class Equation(object):
        def __init__(self, dest, sources):
            self.dest = dest
            self.sources = sources

    class Group(object):
        def __init__(self, equations, real=True, **kw):
            self.equations = equations
            self.real = real

    class MultiStageEquations(object):
        def __init__(self, groups):
            self.groups = groups
    eq.Equation, eq.Group, eq.MultiStageEquations = Equation, Group, MultiStageEquations
    sys.modules['pysph.sph.equation'] = eq
    for mod, cls in (('pysph.sph.integrator_step', 'IntegratorStep'),
                     ('pysph.sph.integrator', 'Integrator'), ('pysph.sph.scheme', 'Scheme')):
        m = types.ModuleType(mod)
        setattr(m, cls, type(cls, (object,), {}))
        if cls == 'Integrator':
            m.IntegratorStep = type('IntegratorStep', (object,), {})
        sys.modules[mod] = m
    ut = types.ModuleType('pysph.base.utils')
    ut.get_particle_array = None
    sys.modules['pysph.base.utils'] = ut
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    _load('pysph.sph.wc.linalg', os.path.join(REF, 'pysph/sph/wc/linalg.py'))
    _load('pysph.sph.wc.viscosity', os.path.join(REF, 'pysph/sph/wc/viscosity.py'))
    crksph = _load('pysph.sph.wc.crksph', os.path.join(REF, 'pysph/sph/wc/crksph.py'))
    return kernels, crksph


def _pair(kernel, d, s, i, j):
    env = pair_symbols(kernel, d, s, i, j)
    XIJ, RIJ = env['XIJ'], env['RIJ']
    hi, hj = d['h'][i], s['h'][j]
    DWI, DWJ = [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]
    kernel.gradient(XIJ, RIJ, hi, DWI)
    kernel.gradient(XIJ, RIJ, hj, DWJ)
    env.update(WI=kernel.kernel(XIJ, RIJ, hi), WJ=kernel.kernel(XIJ, RIJ, hj), DWI=DWI, DWJ=DWJ)
    return env


def refresh(arrays, nreal, dim):
    """every image takes its particle's values (the device's images are the particles)"""
    for a in arrays.values():
        n, ntot = a['_n'], len(a['x'])
        if ntot == n:
            continue
        o = a['orig_idx'][n:].astype(int)
        for p, v in a.items():
            if p in ('x', 'y', 'z', 'tag', 'orig_idx', '_n'):
                continue
            if p in STRIDED:
                st = dim ** STRIDED[p]
                blk = v[:st * ntot].reshape(ntot, st)
                blk[n:] = blk[o]
            else:
                v[n:] = v[o]


def do_group(g, arrays, kernel, nreal, dim):
    k = kernel.radius_scale
    dests = []
    for e in g.equations:
        if e.dest not in dests:
            dests.append(e.dest)
    for dn in dests:
        d = arrays[dn]
        npd = nreal[dn]
        deqs = [e for e in g.equations if e.dest == dn]
        denv = dict(('d_' + p, v) for p, v in d.items())
        denv['SPH_KERNEL'] = kernel
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
            seqs = [e for e in deqs if e.sources and sn in e.sources]
            senv = dict(('s_' + p, v) for p, v in s.items())
            for i in range(npd):
                nb = nbrs(d, s, i, k)
                for j in nb:
                    env = dict(denv, **senv)
                    env.update(_pair(kernel, d, s, i, j))
                    env.update(d_idx=i, s_idx=j)
                    for e in seqs:
                        if hasattr(e, 'loop'):
                            call(e.loop, env)
                for e in seqs:
                    if hasattr(e, 'loop_all'):
                        call(e.loop_all, dict(denv, **senv, d_idx=i, NBRS=nb, N_NBRS=len(nb)))
        for i in range(npd):
            for e in deqs:
                if hasattr(e, 'post_loop'):
                    call(e.post_loop, dict(denv, d_idx=i))
    refresh(arrays, nreal, dim)


def evaluate(groups, arrays, kernel, nreal, dim):
    with np.errstate(divide='ignore', invalid='ignore'):
        for g in groups:
            do_group(g, arrays, kernel, nreal, dim)


def make_case(kind, dim, seed, k, e0, dx=0.1):
    """kind: 'block' (a jittered fluid block), 'rest' (the block at rest: gradv = 0, the limiter's
    0 / 0), 'periodic' (a jittered periodic box).  h varies by +-10 %, rho by +-20 %; e = 0 (p = 0,
    as taylor_green.py runs it) or e0 (1 +- 0.5).  The periodic box takes h = 0.7 dx (k = 2) or
    0.5 dx (k = 3) so that it exceeds twice the support.  Returns (arrays, L)."""
    rs = np.random.RandomState(seed)
    hdx = 1.2
    if kind == 'periodic':
        nfl = {2: (6, 6), 3: (4, 4, 4)}[dim]
        hdx = 0.7 if k == 2 else 0.5
        L = nfl[0] * dx
        pts = lattice(dim, nfl, dx, [0.5 * dx] * 3)
    else:
        nfl = {2: (5, 5), 3: (4, 3, 3)}[dim]
        L = 0.0
        pts = lattice(dim, nfl, dx, [0.0] * 3)
    pts[:, :dim] += rs.uniform(-0.1, 0.1, (len(pts), dim)) * dx
    n = len(pts)
    vel = 0.0 if kind == 'rest' else 1.0
    v = np.zeros((n, 3))
    v[:, :dim] = vel * rs.uniform(-1, 1, (n, dim))
    v0 = v.copy()
    v0[:, :dim] += 0.2 * vel * rs.uniform(-1, 1, (n, dim))
    a = dict(x=pts[:, 0], y=pts[:, 1], z=pts[:, 2], u=v[:, 0], v=v[:, 1], w=v[:, 2],
             u0=v0[:, 0], v0=v0[:, 1], w0=v0[:, 2],
             h=hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)),
             m=dx ** dim * (1.0 + 0.02 * rs.uniform(-1, 1, n)),
             rho=1.0 + 0.2 * rs.uniform(-1, 1, n),
             e=e0 * (1.0 + 0.5 * rs.uniform(-1, 1, n)))
    return dict(fluid=dict((p, _short(x)) for p, x in a.items())), L


def _arrays(inputs, dim, L):
    arrays = {}
    for name, a in inputs.items():
        n = len(a['x'])
        A = dict((p, list(map(float, a.get(p, [0.0] * n)))) for p in PROPS)
        A['tag'] = [0] * n
        A['orig_idx'] = list(range(n))
        if L:
            base = dict((p, list(v)) for p, v in A.items())
            for s in itertools.product((-1, 0, 1), repeat=dim):
                if not any(s):
                    continue
                for p in base:
                    c = 'xyz'.index(p) if p in ('x', 'y', 'z') else -1
                    if 0 <= c < dim and s[c]:
                        A[p] += [x + s[c] * L for x in base[p][:n]]
                    elif p == 'tag':
                        A[p] += [2] * n
                    else:
                        A[p] += list(base[p][:n])
        ntot = len(A['x'])
        A = dict((p, np.array(v, dtype=float)) for p, v in A.items())
        for p in STRIDED:
            A[p] = np.zeros((3 if p in ('bi', 'gradai') else 9) * ntot)
        A['_n'] = n
        arrays[name] = A
    return arrays, dict((nm, a['_n']) for nm, a in arrays.items())


def _out(arrays, props, dim, nreal):
    res = {}
    for nm, a in arrays.items():
        n = nreal[nm]
        res[nm] = {}
        for p in props:
            cnt = n * dim ** STRIDED[p] if p in STRIDED else n
            res[nm][p] = [float('%.15g' % x) for x in a[p][:cnt]]
    return res


def run_case(kernels, crksph, kname, dim, kind, seed, e0=0.0, nu=0.0, g=(0.0, 0.0, 0.0),
             dt=1e-3, steps=0):
    kernel = getattr(kernels, kname)(dim=dim)
    inputs, L = make_case(kind, dim, seed, kernel.radius_scale, e0)
    sch = crksph.CRKSPHScheme(['fluid'], dim, 1.0, 10.0, nu, 0.1, 0.0, gx=g[0], gy=g[1], gz=g[2])
    stages = sch.get_equations().groups
    arrays, nreal = _arrays(inputs, dim, L)
    evaluate(stages[0], arrays, kernel, nreal, dim)
    out0 = _out(arrays, OUT0, dim, nreal)
    evaluate(stages[1], arrays, kernel, nreal, dim)
    out1 = _out(arrays, OUT1, dim, nreal)
    out = dict(kernel=kname, dim=dim, kind=kind, seed=seed, e0=e0, nu=nu, g=list(g), dt=dt, L=L,
               gamma=7.0, inputs=inputs, eval0=out0, eval1=out1, steps=steps)
    if steps:
        # CRKSPHIntegrator from the inputs: initial_acceleration, then `steps` steps (not periodic)
        arrays, nreal = _arrays(inputs, dim, L)
        step = crksph.CRKSPHStep()
        evaluate(stages[0], arrays, kernel, nreal, dim)

        def st(which):
            a = arrays['fluid']
            env = dict([('d_' + p, v) for p, v in a.items()] + [('dt', dt)])
            for i in range(nreal['fluid']):
                call(getattr(step, 'stage%d' % which), dict(env, d_idx=i))
        for _ in range(steps):
            st(1)
            evaluate(stages[0], arrays, kernel, nreal, dim)
            st(2)
            evaluate(stages[1], arrays, kernel, nreal, dim)
            st(3)
        out['stepped'] = _out(arrays, ('x', 'y', 'z', 'u', 'v', 'w', 'e', 'rho', 'p'), dim, nreal)
    return out


# (kernel, dim) -> (geometry, e0, nu, gravity, steps): every kernel in 2-D and 3-D, a fluid at
# rest, e = 0 and e > 0, nu > 0, gravity, a periodic box in 2-D and 3-D, integrator steps
PLAN = {
    ('CubicSpline', 2): ('block', 1.0, 0.0, True, 5),
    ('CubicSpline', 3): ('periodic', 1.0, 0.05, False, 0),
    ('WendlandQuintic', 2): ('rest', 1.0, 0.0, True, 0),
    ('WendlandQuintic', 3): ('block', 0.0, 0.05, False, 0),
    ('QuinticSpline', 2): ('periodic', 0.0, 0.01, False, 0),
    ('QuinticSpline', 3): ('rest', 0.0, 0.0, False, 0),
    ('Gaussian', 2): ('block', 0.0, 0.02, False, 5),
    ('Gaussian', 3): ('block', 1.0, 0.0, True, 0),
}


def gen_cases(kernels, crksph):
    cases = []
    seed = 1200
    for kname in KERNELS:
        for dim in (2, 3):
            seed += 1
            kind, e0, nu, grav, steps = PLAN[kname, dim]
            g = (0.0, 0.0, 0.0) if not grav else \
                ((0.0, -9.81, 0.0) if dim == 2 else (0.0, 0.0, -9.81))
            cases.append(run_case(kernels, crksph, kname, dim, kind, seed, e0=e0, nu=nu, g=g,
                                  steps=steps))
            print(kname, dim, kind, flush=True)
    return cases


def main():
    kernels, crksph = load()
    with open(NAME, 'w') as f:
        json.dump(gen_cases(kernels, crksph), f)
    print('wrote', NAME, os.path.getsize(NAME), 'bytes')


if __name__ == '__main__':
    main()
