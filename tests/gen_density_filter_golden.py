"""Generate tests/golden/density_filter_cases.json FROM THE REFERENCE ITSELF.

TEST INFRASTRUCTURE, run by hand where the reference is present (PYSPH_REFERENCE, default
/root/reference); the fixture it writes is committed.  The reference's
pysph/sph/wc/density_correction.py and pysph/sph/wc/linalg.py are loaded by path, unmodified,
and the initialize / loop_all bodies of ShepardFilter, MLSFirstOrder2D and MLSFirstOrder3D run
on small particle sets, with
  * NBRS by brute force: the sources j of the destination's own array with
    r^2 < (k h_i)^2 or r^2 < (k h_j)^2 (linked_list_nnps.pyx:188), ascending, the particle itself
    included; k the filter kernel's radius scale;
  * the reference's pure-Python kernel objects (pysph/base/kernels.py) as SPH_KERNEL;
  * compyle's `declare` stubbed to zero-filled lists (an int or a tuple of ints for 'int');
  * for MLSFirstOrder3D only, an augmented_matrix that takes its 5-argument call
    augmented_matrix(amls, res, n, 1, aug_mls) as nmax = n: the reference passes the output
    where nmax belongs and raises TypeError; nmax = 4 is what the 2-D body does with n = 3.

    python tests/gen_density_filter_golden.py
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
FILTERS = {'shepard': 'ShepardFilter', 'mls2d_1': 'MLSFirstOrder2D', 'mls3d_1': 'MLSFirstOrder3D'}


def declare(kind, n=1):
    if kind.startswith('matrix'):
        return [0.0] * int(kind[kind.index('(') + 1:kind.index(')')])
    return 0 if n == 1 else (0,) * n


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
    eq.Equation = Equation
    sys.modules['pysph.sph.equation'] = eq
    kernels = _load('pysph.base.kernels', os.path.join(REF, 'pysph/base/kernels.py'))
    linalg = _load('pysph.sph.wc.linalg', os.path.join(REF, 'pysph/sph/wc/linalg.py'))
    dc = _load('pysph.sph.wc.density_correction',
               os.path.join(REF, 'pysph/sph/wc/density_correction.py'))
    return kernels, linalg, dc


def run_filter(kernels, linalg, dc, corr, kernel_name, dim, arrays):
    """One Group([Filter(a, [a])], real=False) per array, as DensityCorrection builds them."""
    kernel = getattr(kernels, kernel_name)(dim=dim)
    cls = getattr(dc, FILTERS[corr])
    aug = linalg.augmented_matrix
    if corr == 'mls3d_1':
        def shim(A, b, n, na, out):
            return aug(A, b, n, na, n, out)
        dc.augmented_matrix = shim
    else:
        dc.augmented_matrix = aug
    k = kernel.radius_scale
    for name, a in arrays.items():
        f = cls(name, [name])
        n = len(a['x'])
        a['rhotmp'] = [0.0] * n
        env = dict(('d_' + p, v) for p, v in a.items())
        env.update(('s_' + p, v) for p, v in a.items())
        for i in range(n):
            call(f.initialize, dict(env, d_idx=i))
        for i in range(n):
            nb = []
            for j in range(n):
                r2 = sum((a[c][i] - a[c][j]) ** 2 for c in 'xyz')
                if r2 < (k * a['h'][i]) ** 2 or r2 < (k * a['h'][j]) ** 2:
                    nb.append(j)
            call(f.loop_all, dict(env, d_idx=i, SPH_KERNEL=kernel, NBRS=nb, N_NBRS=len(nb)))


def lattice(dim, nx, dx, origin):
    axes = [np.arange(nx[d]) * dx + origin[d] for d in range(dim)]
    pts = np.stack([g.ravel() for g in np.meshgrid(*axes, indexing='ij')], axis=1)
    return np.concatenate([pts, np.zeros((len(pts), 3 - dim))], axis=1)


def make_case(dim, seed, dx=0.05, hdx=1.3, rho0=1000.0):
    """A fluid block with a free surface over a wall (truncated support at both), variable h,
    an isolated fluid particle, and in 2-D a vertical line of fluid particles whose
    neighbourhoods are collinear (gj_solve's early return)."""
    rs = np.random.RandomState(seed)
    nxf = (8, 6) if dim == 2 else (5, 4, 4)
    nxw = (8, 2) if dim == 2 else (5, 4, 2)
    fluid = lattice(dim, nxf, dx, [0.0, 0.0, 0.0])
    fluid[:, :dim] += rs.uniform(-0.1, 0.1, (len(fluid), dim)) * dx
    wall = lattice(dim, nxw, dx, [0.0, -2 * dx, 0.0] if dim == 2 else [0.0, 0.0, -2 * dx])
    extra = [[3.0, 3.0, 0.0 if dim == 2 else 3.0]]       # isolated
    if dim == 2:
        extra += [[2.0, 1.0 + 0.5 * k * dx, 0.0] for k in range(4)]   # x_ij = 0 exactly
    fluid = np.concatenate([fluid, np.array(extra)])
    out = {}
    for name, pts in (('fluid', fluid), ('wall', wall)):
        n = len(pts)
        out[name] = dict(
            x=list(map(float, pts[:, 0])), y=list(map(float, pts[:, 1])), z=list(map(float, pts[:, 2])),
            h=list(map(float, hdx * dx * (1.0 + 0.1 * rs.uniform(-1, 1, n)))),
            m=list(map(float, rho0 * dx ** dim * (1.0 + 0.05 * rs.uniform(-1, 1, n)))),
            rho=list(map(float, rho0 * (1.0 + 0.01 * rs.uniform(-1, 1, n)))))
    return out


def gen_density_filter_cases(kernels, linalg, dc):
    cases = []
    seed = 100
    for kname in KERNELS:
        for dim in (2, 3):
            for corr in ('shepard', 'mls2d_1' if dim == 2 else 'mls3d_1'):
                seed += 1
                inputs = make_case(dim, seed)
                arrays = json.loads(json.dumps(inputs))
                run_filter(kernels, linalg, dc, corr, kname, dim, arrays)
                cases.append(dict(kernel=kname, dim=dim, corr=corr, inputs=inputs,
                                  rho=dict((n, a['rho']) for n, a in arrays.items()),
                                  rhotmp=dict((n, a['rhotmp']) for n, a in arrays.items())))
    return cases


def main():
    kernels, linalg, dc = load()
    for m in (dc, linalg):
        m.sqrt, m.abs = math.sqrt, abs
    name = os.path.join(GOLD, 'density_filter_cases.json')
    with open(name, 'w') as f:
        json.dump(gen_density_filter_cases(kernels, linalg, dc), f)
    print('wrote', name, os.path.getsize(name), 'bytes')


if __name__ == '__main__':
    main()
