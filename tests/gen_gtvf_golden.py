"""Generate tests/golden/gtvf_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's pysph/sph/wc/gtvf.py,
transport_velocity.py, linalg.py and pysph/base/kernels.py are loaded by path, unmodified;
GTVFScheme(...).get_equations() gives the two evaluations, and the driver of
tests/gen_iisph_golden.py (acceleration_eval_cython.mako:10-154) runs their bodies, with
SPH_KERNEL the kernel object.  compyle's `declare('matrix(n)')` is a list of n zeros and
`declare('int')` a 0; Equation, Group, MultiStageEquations, Scheme, Integrator and
IntegratorStep are plain bases.  Properties are numpy fp64 arrays, so that CorrectDensity's
m W / rho0 of a wall with rho0 = 0 is inf, as in the compiled reference.

Each case records evaluation 0 and then evaluation 1 on the same inputs; the 2-D wall cases
also record 5 GTVFIntegrator steps (initial_acceleration, then stage1, evaluation 0, stage2,
evaluation 1, stage3).  A periodic case materialises every image of the box as ghost particles
after the real ones (the box exceeds twice the support), as gen_iisph_golden.py does.

    python tests/gen_gtvf_golden.py
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden import REF, GOLD, _load, call, pair_symbols  # noqa: E402
from gen_iisph_golden import lattice, ghosts, nbrs, _short  # noqa: E402

KERNELS = ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
NAME = os.path.join(GOLD, 'gtvf_cases.json')
FLUID_OUT0 = ('arho',)
FLUID_OUT1 = ('rho', 'rhodiv', 'p', 'au', 'av', 'aw', 'auhat', 'avhat', 'awhat', 'p0')
WALL_OUT0 = ('wij', 'ug', 'vg', 'wg')     # (ug = 2 u - uf checks uf too)
WALL_OUT1 = ('V', 'p', 'wij', 'rho')
PROPS = ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'p', 'au', 'av', 'aw', 'uhat', 'vhat',
         'what', 'rho0', 'rhodiv', 'p0', 'auhat', 'avhat', 'awhat', 'arho', 'arho0', 'uf', 'vf',
         'wf', 'ug', 'vg', 'wg', 'wij', 'V', 'tag', 'orig_idx')


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
        sys.modules[mod] = m
    ut = types.ModuleType('pysph.base.utils')
    ut.get_particle_array = None
    sys.modules['pysph.base.utils'] = ut
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    _load('pysph.sph.wc.linalg', os.path.join(REF, 'pysph/sph/wc/linalg.py'))
    _load('pysph.sph.wc.transport_velocity', os.path.join(REF, 'pysph/sph/wc/transport_velocity.py'))
    gtvf = _load('pysph.sph.wc.gtvf', os.path.join(REF, 'pysph/sph/wc/gtvf.py'))
    return kernels, gtvf


def do_group(g, arrays, kernel, nreal, dt):
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
        denv.update(dt=dt, SPH_KERNEL=kernel)
        for i in range(npd):
            for e in deqs:
                if hasattr(e, 'initialize'):
                    call(e.initialize, dict(denv, d_idx=i))
        srcs = []
        for e in deqs:
            for s in (e.sources or []):
                if s not in srcs:
                    srcs.append(s)
        for i in range(npd):
            for e in deqs:
                if e.sources is None and hasattr(e, 'loop'):
                    call(e.loop, dict(denv, d_idx=i))
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


def evaluate(groups, arrays, kernel, nreal, dt):
    with np.errstate(divide='ignore', invalid='ignore'):
        for g in groups:
            do_group(g, arrays, kernel, nreal, dt)


def make_case(kind, dim, seed, k, dx=0.1):
    """kind: 'tank' (a jittered fluid block with a free surface over a 4-layer wall), 'block'
    (the block alone), 'periodic' (a jittered periodic box).  h varies by +-10 %, rho by +-40 %
    (so that both branches of min(10 |p|, pref) occur).  k: the kernel's radius scale; the periodic
    box takes h = 0.7 dx (k = 2) or 0.5 dx (k = 3), as gen_iisph_golden.py does, so that it exceeds
    twice the support.  In 3-D the wall lies under the block only.  Returns (arrays, fluids,
    solids, L)."""
    rs = np.random.RandomState(seed)
    hdx = 1.2

    def arr(pts, vel, rho_var):
        n = len(pts)
        v = np.zeros((n, 3))
        v[:, :dim] = vel * rs.uniform(-1, 1, (n, dim))
        vh = v.copy()
        vh[:, :dim] += 0.2 * vel * rs.uniform(-1, 1, (n, dim))
        a = dict(x=pts[:, 0], y=pts[:, 1], z=pts[:, 2], u=v[:, 0], v=v[:, 1], w=v[:, 2],
                 uhat=vh[:, 0], vhat=vh[:, 1], what=vh[:, 2],
                 h=hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)),
                 m=1000.0 * dx ** dim * (1.0 + 0.02 * rs.uniform(-1, 1, n)),
                 rho=1000.0 * (1.0 + rho_var * rs.uniform(-1, 1, n)),
                 au=vel * rs.uniform(-1, 1, n), av=vel * rs.uniform(-1, 1, n),
                 auhat=vel * rs.uniform(-1, 1, n), avhat=vel * rs.uniform(-1, 1, n))
        if dim == 3:
            a.update(aw=vel * rs.uniform(-1, 1, n), awhat=vel * rs.uniform(-1, 1, n))
        return dict((p, _short(x)) for p, x in a.items())
    if kind == 'periodic':
        nfl = {2: (6, 6), 3: (5, 5, 5)}[dim]
        hdx = 0.7 if k == 2 else 0.5
        L = nfl[0] * dx
        pts = lattice(dim, nfl, dx, [0.5 * dx] * 3)
        pts[:, :dim] += rs.uniform(-0.1, 0.1, (len(pts), dim)) * dx
        f = arr(pts, 1.0, 0.4)
        f['rho0'] = list(f['rho'])
        return dict(fluid=f), ['fluid'], [], L
    nfl = {2: (5, 4), 3: (3, 3, 3)}[dim]
    pts = lattice(dim, nfl, dx, [0.0] * 3)
    pts[:, :dim] += rs.uniform(-0.1, 0.1, (len(pts), dim)) * dx
    arrays = dict(fluid=arr(pts, 1.0, 0.4))
    solids = []
    if kind.startswith('tank'):
        wn = (nfl[0] + 2, 4) if dim == 2 else (nfl[0], nfl[1], 4)
        wall = lattice(dim, wn, dx, [-dx, -4.0 * dx, 0.0] if dim == 2 else [0.0, 0.0, -4.0 * dx])
        w = arr(wall, 0.0, 0.0)
        w['u'] = [0.1] * len(w['x'])        # a moving wall: ug differs from -uf
        w['au'] = [0.5] * len(w['x'])       # a prescribed wall acceleration (SolidWallPressureBC)
        # dam_break_2d.py leaves the walls' rho0 at 0 (setup_properties adds it); 'tank_rho'
        # gives them rho0 = rho
        w['rho0'] = list(w['rho']) if kind == 'tank_rho' else [0.0] * len(w['x'])
        arrays['wall'] = w
        solids = ['wall']
    return arrays, ['fluid'], solids, 0.0


def _arrays(inputs, dim, L):
    arrays = json.loads(json.dumps(inputs))
    for a in arrays.values():
        n = len(a['x'])
        for p in PROPS:
            a.setdefault(p, [0.0] * n)
    nreal = ghosts(arrays, dim, L)
    out = dict((nm, dict((p, np.array(v, dtype=float)) for p, v in a.items()))
               for nm, a in arrays.items())
    for a in out.values():                  # stride 9 (GTVFStep.stage2 adds dt asigma = 0)
        a['sigma'], a['asigma'] = np.zeros(9 * len(a['x'])), np.zeros(9 * len(a['x']))
    return out, nreal


def _out(arrays, names, nreal, fluids, solids, fo, wo, prefix=''):
    res = {}
    for nm in names:
        props = fo if nm in fluids else wo
        res[nm] = dict((prefix + p, [float('%.15g' % x) for x in arrays[nm][p][:nreal[nm]]]) for p in props)
    return res


def run_case(kernels, gtvf, kname, dim, kind, seed, pref, alpha=0.0, nu=0.0, g=(0.0, 0.0, 0.0),
             dt=1e-3, steps=0):
    kernel = getattr(kernels, kname)(dim=dim)
    inputs, fluids, solids, L = make_case(kind, dim, seed, kernel.radius_scale)
    sch = gtvf.GTVFScheme(fluids, solids, dim, 1000.0, 10.0, nu, None, pref, gx=g[0], gy=g[1],
                          gz=g[2], alpha=alpha)
    stages = sch.get_equations().groups
    arrays, nreal = _arrays(inputs, dim, L)
    evaluate(stages[0], arrays, kernel, nreal, dt)
    out0 = _out(arrays, fluids + solids, nreal, fluids, solids, FLUID_OUT0, WALL_OUT0)
    evaluate(stages[1], arrays, kernel, nreal, dt)
    out1 = _out(arrays, fluids + solids, nreal, fluids, solids, FLUID_OUT1, WALL_OUT1)
    out = dict(kernel=kname, dim=dim, kind=kind, seed=seed, pref=pref, alpha=alpha, nu=nu, c0=10.0,
               g=list(g), dt=dt, L=L, rho0=1000.0, fluids=fluids, solids=solids, inputs=inputs,
               eval0=out0, eval1=out1, steps=steps)
    if steps:
        # GTVFIntegrator from the inputs: initial_acceleration, then `steps` steps
        arrays, nreal = _arrays(inputs, dim, L)
        step = gtvf.GTVFStep()
        evaluate(stages[0], arrays, kernel, nreal, dt)

        def st(which):
            for f in fluids:
                a = arrays[f]
                for i in range(nreal[f]):
                    call(getattr(step, 'stage%d' % which),
                         dict([('d_' + p, v) for p, v in a.items()] + [('d_idx', i), ('dt', dt)]))
        for _ in range(steps):
            st(1)
            evaluate(stages[0], arrays, kernel, nreal, dt)
            st(2)
            evaluate(stages[1], arrays, kernel, nreal, dt)
            st(3)
        out['stepped'] = _out(arrays, fluids + solids, nreal, fluids, solids,
                              ('x', 'y', 'z', 'u', 'v', 'w', 'rho', 'p'), ('rho', 'p'))
    return out


# (kernel, dim) -> (geometry, alpha, nu, steps): every geometry in 2-D and 3-D, a wall with
# rho0 = 0 and one with rho0 = rho, alpha > 0 beside walls, nu > 0 in the periodic box
PLAN = {
    ('CubicSpline', 2): ('tank', 0.1, 0.0, 5),
    ('CubicSpline', 3): ('periodic', 0.0, 0.05, 0),
    ('WendlandQuintic', 2): ('tank_rho', 0.0, 0.0, 5),
    ('WendlandQuintic', 3): ('tank', 0.1, 0.0, 0),
    ('QuinticSpline', 2): ('periodic', 0.0, 0.02, 0),
    ('QuinticSpline', 3): ('tank_rho', 0.2, 0.0, 0),
    ('Gaussian', 2): ('block', 0.1, 0.01, 0),
    ('Gaussian', 3): ('tank', 0.0, 0.0, 0),
}


def gen_cases(kernels, gtvf):
    cases = []
    seed = 900
    for kname in KERNELS:
        for dim in (2, 3):
            seed += 1
            kind, alpha, nu, steps = PLAN[kname, dim]
            g = (0.0, 0.0, 0.0) if kind in ('block', 'periodic') else \
                ((0.0, -9.81, 0.0) if dim == 2 else (0.0, 0.0, -9.81))
            cases.append(run_case(kernels, gtvf, kname, dim, kind, seed, pref=1000.0 * 100.0,
                                  alpha=alpha, nu=nu, g=g, steps=steps))
            print(kname, dim, kind, flush=True)
    return cases


def main():
    kernels, gtvf = load()
    with open(NAME, 'w') as f:
        json.dump(gen_cases(kernels, gtvf), f)
    print('wrote', NAME, os.path.getsize(NAME), 'bytes')


if __name__ == '__main__':
    main()
