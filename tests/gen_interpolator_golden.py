"""Generate tests/golden/interpolator_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's pysph/tools/interpolator.py,
pysph/sph/basic_equations.py and pysph/sph/wc/linalg.py are loaded by path, unmodified (their
imports of the compiled machinery are stubbed), and the bodies of InterpolateFunction,
InterpolateSPH, SPLASHInterpolateProperty, SPLASHInterpolatePropertyNormalized, SummationDensity,
SPHFirstOrderApproximationPreStep and SPHFirstOrderApproximation run over a brute-force fp64
neighbour loop in the order the Interpolator's Groups run them:
  * neighbours of a destination: every source with r^2 < (k h_d)^2 or r^2 < (k h_s)^2
    (linked_list_nnps.pyx:188), k the interpolation kernel's radius scale;
  * WIJ, WI, WJ, DWIJ from the reference's pure-Python kernel objects at HIJ = (h_d + h_s) / 2, h_d
    and h_s;
  * sources: every particle of every array, ghosts included; in a periodic box, the images of
    every particle within one box length are materialised (the oracle's way) and the probes are
    wrapped into the box first (_box_wrap_periodic, nnps_base.pyx:699-743);
  * an array that lacks the property gives temp_prop = 0 (interpolator.py:360-366);
  * order1: SummationDensity over all sources (Group real=False) first, its rho used by the
    next two Groups.

    python tests/gen_interpolator_golden.py
"""
import json
import math
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.gen_golden import REF, GOLD, _load, call  # noqa: E402

KERNELS = ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
METHODS = ('shepard', 'sph', 'splash', 'splash_norm', 'order1')
NAMES = ('fluid', 'solid')


def declare(kind, n=1):
    if kind.startswith('matrix'):
        return [0.0] * int(kind[kind.index('(') + 1:kind.index(')')])
    return 0 if n == 1 else (0,) * n


def load():
    for pkg in ('pysph', 'pysph.sph', 'pysph.sph.wc', 'pysph.base', 'pysph.tools', 'compyle'):
        sys.modules.setdefault(pkg, types.ModuleType(pkg))
    api = types.ModuleType('compyle.api')
    api.declare = declare
    sys.modules['compyle.api'] = api
    eq = types.ModuleType('pysph.sph.equation')

    class Equation(object):
        def __init__(self, dest, sources):
            self.dest = dest
            self.sources = sources
    eq.Equation = Equation
    eq.Group = object
    sys.modules['pysph.sph.equation'] = eq
    # what interpolator.py imports of the compiled machinery: unused by the bodies
    for name, attrs in (('pysph.base.utils', ('get_particle_array',)),
                        ('pysph.base.nnps', ('LinkedListNNPS',)),
                        ('pysph.sph.acceleration_eval', ('AccelerationEval',)),
                        ('pysph.sph.sph_compiler', ('SPHCompiler',))):
        m = types.ModuleType(name)
        for a in attrs:
            setattr(m, a, None)
        sys.modules[name] = m
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    linalg = _load('pysph.sph.wc.linalg', os.path.join(REF, 'pysph/sph/wc/linalg.py'))
    basic = _load('pysph.sph.basic_equations', os.path.join(REF, 'pysph/sph/basic_equations.py'))
    interp = _load('pysph.tools.interpolator', os.path.join(REF, 'pysph/tools/interpolator.py'))
    for m in (linalg, interp):
        m.abs = abs
    return kernels, basic, interp


def images(src, box):
    """the sources and, in a periodic box, their images within one box length per axis"""
    if box is None:
        return src
    lo, hi, per = np.array(box['lo']), np.array(box['hi']), box['periodic']
    L = hi - lo
    shifts = [np.zeros(3)]
    for d in range(3):
        if per[d]:
            shifts = [s + e * L[d] * np.eye(3)[d] for s in shifts for e in (-1, 0, 1)]
    out = dict((k, []) for k in src)
    for s in shifts:
        for k in src:
            v = np.array(src[k])
            if k in 'xyz':
                v = v + s['xyz'.index(k)]
            out[k].append(v)
    return dict((k, np.concatenate(v)) for k, v in out.items())


def wrap(p, box):
    p = np.array(p, dtype=float)
    if box is None:
        return p
    for d in range(3):
        if box['periodic'][d]:
            lo, hi = box['lo'][d], box['hi'][d]
            L = hi - lo
            p[d] = np.where(p[d] < lo, p[d] + L, p[d])
            p[d] = np.where(p[d] > hi, p[d] - L, p[d])
    return p


def run(kernels, basic, interp, kname, dim, method, case):
    kernel = getattr(kernels, kname)(dim=dim)
    k = kernel.radius_scale
    box = case.get('box')
    # every source particle of every array; temp_prop = f or 0
    src = dict((c, []) for c in ('x', 'y', 'z', 'h', 'm', 'rho', 'temp_prop'))
    for name in NAMES:
        a = case['arrays'][name]
        for c in ('x', 'y', 'z', 'h', 'm', 'rho'):
            src[c] += a[c]
        src['temp_prop'] += a['f'] if 'f' in a else [0.0] * len(a['x'])
    src = images(src, box)
    src = dict((c, list(map(float, v))) for c, v in src.items())
    ns = len(src['x'])
    P = wrap([case['probes'][c] for c in 'xyz'], box)
    npb = P.shape[1]
    hp = max(max(case['arrays'][n]['h']) for n in NAMES)
    d = dict(x=list(P[0]), y=list(P[1]), z=list(P[2]), h=[hp] * npb, number_density=[0.0] * npb,
             prop=[0.0] * (npb * (4 if method == 'order1' else 1)), unity=[0.0] * npb,
             moment=[0.0] * (16 * npb), p_sph=[0.0] * (4 * npb))
    pos = np.array([src['x'], src['y'], src['z']]).T

    def nbrs(q, hq):
        r2 = np.sum((pos - q) ** 2, axis=1)
        return [j for j in range(ns) if r2[j] < (k * hq) ** 2 or r2[j] < (k * src['h'][j]) ** 2]

    def pair_env(di, dd, j):
        xij = [dd['x'][di] - src['x'][j], dd['y'][di] - src['y'][j], dd['z'][di] - src['z'][j]]
        rij = math.sqrt(sum(v * v for v in xij))
        hd, hs = dd['h'][di], src['h'][j]
        hij = 0.5 * (hd + hs)
        dwij = [0.0, 0.0, 0.0]
        kernel.gradient(xij, rij, hij, dwij)
        env = dict(('d_' + p, v) for p, v in dd.items())
        env.update(('s_' + p, v) for p, v in src.items())
        env.update(d_idx=di, s_idx=j, XIJ=xij, RIJ=rij, HIJ=hij, DWIJ=dwij,
                   WIJ=kernel.kernel(xij, rij, hij), WI=kernel.kernel(xij, rij, hd),
                   WJ=kernel.kernel(xij, rij, hs))
        return env

    def group(eq, dd, nd):
        env0 = dict(('d_' + p, v) for p, v in dd.items())
        for i in range(nd):
            if hasattr(eq, 'initialize'):
                call(eq.initialize, dict(env0, d_idx=i))
        for i in range(nd):
            q = np.array([dd['x'][i], dd['y'][i], dd['z'][i]])
            for j in nbrs(q, dd['h'][i]):
                call(eq.loop, pair_env(i, dd, j))
        for i in range(nd):
            if hasattr(eq, 'post_loop'):
                call(eq.post_loop, dict(env0, d_idx=i))

    cls = {'shepard': interp.InterpolateFunction, 'sph': interp.InterpolateSPH,
           'splash': interp.SPLASHInterpolateProperty,
           'splash_norm': interp.SPLASHInterpolatePropertyNormalized}
    if method in cls:
        group(cls[method]('interpolate', list(NAMES)), d, npb)
    else:
        sd = dict(src)
        sd['rho'] = list(sd['rho'])
        group(basic.SummationDensity('sources', ['sources']), sd, ns)
        src['rho'] = sd['rho']
        group(interp.SPHFirstOrderApproximationPreStep('interpolate', list(NAMES), dim=dim), d, npb)
        group(interp.SPHFirstOrderApproximation('interpolate', list(NAMES), dim=dim), d, npb)
    return d['prop']


def lattice(dim, nx, dx, origin):
    axes = [np.arange(nx[d]) * dx + origin[d] for d in range(dim)]
    pts = np.stack([g.ravel() for g in np.meshgrid(*axes, indexing='ij')], axis=1)
    return np.concatenate([pts, np.zeros((len(pts), 3 - dim))], axis=1)


def make_case(dim, seed, periodic=False, dx=0.1, hdx=1.3):
    """A jittered fluid block with variable h and a field f, a solid layer that lacks f, an
    isolated fluid particle; probes inside the cloud, far outside it (zero weight), next to the
    isolated particle, and, in 2-D, on a line of fluid particles with x_ij = 0 (collinear
    neighbourhood: order1's gj_solve returns early).  periodic: a box around the block along
    x, with probes outside it."""
    rs = np.random.RandomState(seed)
    nxf = {1: (10,), 2: (20, 6) if periodic else (8, 6), 3: (5, 4, 4)}[dim]
    nxs = {1: (3,), 2: (20, 2) if periodic else (8, 2), 3: (5, 4, 2)}[dim]
    fluid = lattice(dim, nxf, dx, [0.0, 0.0, 0.0])
    fluid[:, :dim] += rs.uniform(-0.1, 0.1, (len(fluid), dim)) * dx
    so = [-3 * dx, 0.0, 0.0] if dim == 1 else ([0.0, -2 * dx, 0.0] if dim == 2 else [0.0, 0.0, -2 * dx])
    solid = lattice(dim, nxs, dx, so)
    far = [30.0, 0.0, 0.0] if dim == 1 else ([30.0, 30.0, 0.0] if dim == 2 else [30.0, 30.0, 30.0])
    extra = [far]                                            # isolated
    if dim == 2:
        extra += [[5.0, 1.0 + 0.5 * k * dx, 0.0] for k in range(4)]   # x_ij = 0 exactly
    fluid = np.concatenate([fluid, np.array(extra)])
    arrays = {}
    for name, pts in (('fluid', fluid), ('solid', solid)):
        n = len(pts)
        a = dict(x=pts[:, 0], y=pts[:, 1], z=pts[:, 2],
                 h=hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)),
                 m=dx ** dim * (1.0 + 0.05 * rs.uniform(-1, 1, n)),
                 rho=1.0 + 0.01 * rs.uniform(-1, 1, n))
        if name == 'fluid':
            a['f'] = np.sin(2.0 * pts[:, 0]) + pts[:, 1] - 0.5 * pts[:, 2] + 2.0
        arrays[name] = dict((k, list(map(float, v))) for k, v in a.items())
    ext = np.array(nxf + (1,) * (3 - dim)) * dx
    inside = rs.uniform(0.1, 0.9, (8, 3)) * ext
    inside[:, dim:] = 0.0
    probes = list(inside) + [np.array([-20.0, -20.0, -20.0])[:3] * (np.arange(3) < dim),
                             np.array(far) + 0.3 * dx * (np.arange(3) < dim)]
    if dim == 2:
        probes += [np.array([5.0, 1.0 + 0.75 * dx, 0.0])]
    case = dict(arrays=arrays)
    if periodic:
        lo = [-0.5 * dx, -1e3, -1e3]
        hi = [nxf[0] * dx - 0.5 * dx, 1e3, 1e3]
        case['box'] = dict(lo=lo, hi=hi, periodic=[True, False, False])
        # only the block and the solid (the far particles would leave the box)
        arrays['fluid'] = dict((k, v[:int(np.prod(nxf))]) for k, v in arrays['fluid'].items())
        probes = list(inside) + [np.array([hi[0] + 0.3 * dx, inside[0][1], inside[0][2]]),
                                 np.array([lo[0] - 2.2 * dx, inside[1][1], inside[1][2]])]
    P = np.array(probes)
    case['probes'] = dict(x=list(map(float, P[:, 0])), y=list(map(float, P[:, 1])),
                          z=list(map(float, P[:, 2])))
    return case


def gen_cases(kernels, basic, interp):
    cases = []
    seed = 200
    for kname in KERNELS:
        for dim in (1, 2, 3):
            if kname == 'WendlandQuintic' and dim == 1:
                continue
            for periodic in ((False, True) if dim == 2 else (False,)):
                seed += 1
                case = make_case(dim, seed, periodic=periodic)
                case.update(kernel=kname, dim=dim, periodic=periodic, results={})
                for method in METHODS:
                    case['results'][method] = run(kernels, basic, interp, kname, dim, method,
                                                  json.loads(json.dumps(case)))
                cases.append(case)
    return cases


def main():
    kernels, basic, interp = load()
    name = os.path.join(GOLD, 'interpolator_cases.json')
    with open(name, 'w') as f:
        json.dump(gen_cases(kernels, basic, interp), f)
    print('wrote', name, os.path.getsize(name), 'bytes')


if __name__ == '__main__':
    main()
