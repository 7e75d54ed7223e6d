"""Generate tests/golden/shift_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's pysph/sph/wc/shift.py and
pysph/base/kernels.py are loaded by path, unmodified, and ShiftPositions' Groups run on small
particle sets:
  * Group([SimpleShift(a, [a], const)]) or Group([FickianShift(a, [a], fickian_const, ...)]):
    SimpleShift.py_initialize, then loop_all for every real particle of the array, with NBRS by
    brute force -- the sources j of the array itself (periodic images materialised) with
    r^2 < (k h_i)^2 or r^2 < (k h_j)^2 (linked_list_nnps.pyx:188), ascending, the particle
    itself included.  s_x / s_y / s_z are bound to a copy frozen before the shift: the device
    forms every dpos from the positions before the shift (a Jacobi update);
  * with the correction, NBRS again from the shifted positions, then CorrectVelocities'
    initialize, loop (DWIJ, VIJ as oracle/gen_golden.py forms them) and post_loop;
  * compyle's `declare` stubbed to zero-filled lists, serial_reduce_array to numpy and
    parallel_reduce_array to the identity; Equation and Tool to plain bases.
Every case also records N_NBRS per particle.  The second array ('wall') is never a source.

    python tests/gen_shift_golden.py
"""
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
NAME = os.path.join(GOLD, 'shift_cases.json')


def declare(kind, n=1):
    if kind.startswith('matrix'):
        size = int(kind[kind.index('(') + 1:kind.index(')')])
        return [0.0] * size if n == 1 else tuple([0.0] * size for _ in range(n))
    return 0 if n == 1 else (0,) * n


def load():
    for pkg in ('pysph', 'pysph.sph', 'pysph.sph.wc', 'pysph.base', 'pysph.solver', 'compyle'):
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
    sys.modules['pysph.sph.equation'] = eq
    ra = types.ModuleType('pysph.base.reduce_array')
    ra.serial_reduce_array = lambda a, op: getattr(np, op)(a)
    ra.parallel_reduce_array = lambda a, op: a
    sys.modules['pysph.base.reduce_array'] = ra
    tools = types.ModuleType('pysph.solver.tools')
    tools.Tool = type('Tool', (object,), {})
    sys.modules['pysph.solver.tools'] = tools
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    shift = _load('pysph.sph.wc.shift', os.path.join(REF, 'pysph/sph/wc/shift.py'))
    return kernels, shift


def sources(a, dim, L):
    """the array's particles and, in a periodic box of edge L (every axis < dim), their images
    x + s L, s in {-1, 0, 1}^dim \\ 0, as lists; and the index of each source's particle"""
    n = len(a['x'])
    shifts = [(0, 0, 0)]
    if L:
        import itertools
        shifts += [s + (0,) * (3 - dim) for s in itertools.product((-1, 0, 1), repeat=dim)
                   if any(s)]
    out = dict((p, []) for p in a)
    owner = []
    for s in shifts:
        for p in a:
            v = a[p]
            if p in 'xyz':
                d = 'xyz'.index(p)
                out[p] += [v[i] + s[d] * L for i in range(n)] if s[d] else list(v)
            else:
                out[p] += list(v)
        owner += list(range(n))
    return out, owner


def nbrs(a, src, owner, i, k):
    """the brute-force NBRS of destination i, ascending by particle then image; r^2 formed as
    the neighbour search forms it (norm2(s_x - x, ..), linked_list_nnps.pyx:183-185)"""
    d = [np.array(src[c]) - a[c][i] for c in 'xyz']
    r2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    hi = k * a['h'][i]
    hj = k * np.array(src['h'])
    ok = (r2 < hi * hi) | (r2 < hj * hj)
    return sorted(map(int, np.nonzero(ok)[0]), key=lambda j: (owner[j], j))


def run_tool(kernels, shift, kname, dim, kind, const, correct, a, L, tensile=False, dt=1e-3):
    """ShiftPositions' Groups on array `a` (dict of lists, changed in place).  Returns dpos,
    N_NBRS of the shift and, with the correction, N_NBRS of the correction."""
    kernel = getattr(kernels, kname)(dim=dim)
    k = kernel.radius_scale
    n = len(a['x'])
    a['dpos'] = [0.0] * (3 * n)
    if kind == 'simple':
        eq = shift.SimpleShift('fluid', ['fluid'], const=const)
        dst = types.SimpleNamespace(**dict((p, np.array(a[p])) for p in 'uvw'))
        dst.vmax = np.zeros(1)
        eq.py_initialize(dst, 0.0, dt)
        a['vmax'] = [float(dst.vmax[0])]
    else:
        eq = shift.FickianShift('fluid', ['fluid'], fickian_const=const,
                                tensile_correction=tensile)
    frozen = json.loads(json.dumps(a))
    src, owner = sources(frozen, dim, L)
    nn = []
    for i in range(n):
        nb = nbrs(frozen, src, owner, i, k)
        nn.append(len(nb))
        env = dict(('d_' + p, v) for p, v in a.items())
        env.update(('s_' + p, v) for p, v in src.items())
        env.update(d_idx=i, dt=dt, NBRS=nb, N_NBRS=len(nb), SPH_KERNEL=kernel)
        call(eq.loop_all, env)
    out = dict(dpos=list(a['dpos']), n_nbrs=nn)
    if correct:
        cv = shift.CorrectVelocities('fluid', ['fluid'])
        a['gradv'] = [0.0] * (9 * n)
        src, owner = sources(a, dim, L)
        nn = []
        for i in range(n):
            call(cv.initialize, dict(d_idx=i, d_gradv=a['gradv']))
        for i in range(n):
            nb = nbrs(a, src, owner, i, k)
            nn.append(len(nb))
            for j in nb:
                env = pair_symbols(kernel, a, src, i, j)
                env.update(d_idx=i, s_idx=j, s_m=src['m'], s_rho=src['rho'], d_gradv=a['gradv'])
                call(cv.loop, env)
        for i in range(n):
            call(cv.post_loop, dict(d_idx=i, d_u=a['u'], d_v=a['v'], d_w=a['w'], d_gradv=a['gradv'],
                                    d_dpos=a['dpos']))
        out['n_nbrs_correct'] = nn
    return out


def lattice(dim, nx, dx, origin):
    axes = [np.arange(nx[d]) * dx + origin[d] for d in range(dim)]
    pts = np.stack([g.ravel() for g in np.meshgrid(*axes, indexing='ij')], axis=1)
    return np.concatenate([pts, np.zeros((len(pts), 3 - dim))], axis=1)


def _short(v):
    """inputs with 6 significant digits: the fixture stays small, and the reference runs on
    exactly the values it records"""
    return [float('%.6g' % x) for x in v]


def make_case(dim, seed, k, periodic, dx=0.1):
    """A jittered block with a free surface, an isolated particle and a particle at rest; or a
    jittered periodic lattice whose edge L exceeds twice the largest support (a pair meets one
    image at most).  h varies by +-10 %.  Beside it a row of wall particles that is never a
    source.  No pair lies within 1e-9 (relative) of the accept radius: the seed is advanced
    until none does.  Returns (arrays, L, seed)."""
    if periodic:
        nx = {1: (12,), 2: (5, 5), 3: (4, 4, 4)}[dim]
        hdx = {1: 1.0, 2: 1.0 if k == 2 else 0.7, 3: 0.9 if k == 2 else 0.6}[dim]
        origin, L = [0.5 * dx] * 3, nx[0] * dx
    else:
        nx = {1: (10,), 2: (6, 5), 3: (3, 3, 3)}[dim]
        hdx, origin, L = 1.0, [0.0] * 3, 0.0
    while True:
        rs = np.random.RandomState(seed)
        fluid = lattice(dim, nx, dx, origin)
        fluid[:, :dim] += rs.uniform(-0.15, 0.15, (len(fluid), dim)) * dx
        if not periodic:
            fluid = np.concatenate([fluid, [[5.0, 5.0 if dim > 1 else 0.0, 5.0 if dim > 2 else 0.0]]])
        n = len(fluid)
        vel = np.zeros((n, 3))
        vel[:, :dim] = rs.uniform(-1, 1, (n, dim))
        vel[0] = 0.0                                     # a particle at rest
        a = dict(x=fluid[:, 0], y=fluid[:, 1], z=fluid[:, 2], u=vel[:, 0], v=vel[:, 1], w=vel[:, 2],
                 h=hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)),
                 m=1000.0 * dx ** dim * (1.0 + 0.05 * rs.uniform(-1, 1, n)),
                 rho=1000.0 * (1.0 + 0.01 * rs.uniform(-1, 1, n)))
        a = dict((p, _short(v)) for p, v in a.items())
        pos = np.stack([a[c] for c in 'xyz'], axis=1)
        h = np.array(a['h'])
        ok = True
        for i in range(n):
            d = pos - pos[i]
            if periodic:
                d[:, :dim] -= L * np.round(d[:, :dim] / L)
            r = np.sqrt(np.sum(d * d, axis=1))
            for lim in (k * h[i], k * h):
                if np.any(np.abs(r - lim) <= 1e-9 * lim):
                    ok = False
        if ok:
            break
        seed += 1000
    wall = lattice(dim, (nx[0],) + (1,) * (dim - 1), dx, [0.0, -2 * dx, 0.0] if dim == 2 else
                   [0.0, 0.0, -2 * dx] if dim == 3 else [-3 * dx, 0.0, 0.0])
    nw = len(wall)
    w = dict(x=wall[:, 0], y=wall[:, 1], z=wall[:, 2], u=np.full(nw, 0.3), v=np.zeros(nw),
             w=np.zeros(nw), h=np.full(nw, hdx * dx), m=np.full(nw, 1000.0 * dx ** dim),
             rho=np.full(nw, 1000.0))
    return dict(fluid=a, wall=dict((p, _short(v)) for p, v in w.items())), L, seed


def gen_cases(kernels, shift, only=None):
    """Every kernel in 1-3 D (WendlandQuintic not in 1-D) x {simple, fickian} x {correct, not}.
    A kind shifts a periodic box with the correction and the block without it, or the other
    way round, so that each kind and the correction see both geometries.  FickianShift with
    the correction runs with tensile_correction in 2-D.  Every other case gives the tool's
    `parameter`, the rest take its default.  The shifted positions are the inputs plus dpos
    (the reference's d_x += d_dpos); u, v, w are recorded after a correction.  Returns every
    case, or only those whose index is in `only` (None for the others)."""
    cases = []
    seed = 300
    for kname in KERNELS:
        k = getattr(kernels, kname)(dim=2).radius_scale
        for dim in (1, 2, 3):
            if kname == 'WendlandQuintic' and dim == 1:
                continue
            for kind in ('simple', 'fickian'):
                for correct in (False, True):
                    seed += 1
                    if only is not None and len(cases) not in only:
                        cases.append(None)
                        continue
                    periodic = (kind == 'simple') == correct
                    parameter = None if seed % 2 else (0.1 if kind == 'simple' else 2.5)
                    const = parameter or (0.04 if kind == 'simple' else 4)
                    tensile = kind == 'fickian' and correct and dim == 2
                    inputs, L, used = make_case(dim, seed, k, periodic)
                    a = json.loads(json.dumps(inputs['fluid']))
                    res = run_tool(kernels, shift, kname, dim, kind, const, correct, a, L,
                                   tensile=tensile)
                    for d, c in enumerate('xyz'):
                        assert a[c] == [x + dp for x, dp in zip(inputs['fluid'][c], res['dpos'][d::3])]
                    if correct:
                        res.update(u=a['u'], v=a['v'], w=a['w'])
                    cases.append(dict(kernel=kname, dim=dim, kind=kind, correct=correct,
                                      parameter=parameter, const=const, tensile=tensile, dt=1e-3,
                                      L=L, seed=used, inputs=inputs, vmax=a.get('vmax'), **res))
    return cases


def main():
    kernels, shift = load()
    shift.sqrt = math.sqrt
    with open(NAME, 'w') as f:
        json.dump(gen_cases(kernels, shift), f)
    print('wrote', NAME, os.path.getsize(NAME), 'bytes')


if __name__ == '__main__':
    main()
