"""k_tvf_pass1, k_tvf_wall and k_tvf_pass2 (plain, WALLS, EXT) -- the EDAC scheme -- against the
fp64 oracle.

test_gpu_edac.py compares one evaluation with three sets of four small reference-generated cases
(at most four of the eleven (kernel, dim) pairs each, never Gaussian or 1-D) and Taylor-Green
runs.  Here one b200sph_tvf_pass runs, for every (kernel, dim) the kernels are instantiated for,
against the oracle's passes in the order program.py emits them, for the internal flow without
walls, with solid walls and the external flow (pb = 0, with and without ClampWallPressure), on
two fluid arrays (trailing particles of the first are ghosts) and two wall arrays (the second
with a prescribed acceleration), with alpha, nu and a separate edac_nu != 0, gravity along
every axis, damped (t < tdamp) or not, with and without the average pressure.  The geometry is
the one of the WCSPH pair-kernel test (a jittered lattice, a double-density cluster, a sparse
corner, a coincident pair, an isolated fluid particle) plus a wall particle with no fluid
neighbour, with h varying by +-20 %, large enough for several CTAs.  test_edac_oracle_on_cpu.py
runs the same checks on the library emulation.
"""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import rel_err
from oracle import oracle as orc
from test_gpu_parity import TOL_EVAL
from test_gpu_records32_oracle import KERNEL_DIMS, _positions
from test_gpu_solid_oracle import _fix_h

pytestmark = pytest.mark.gpu

NAMES = ('fluid_a', 'fluid_b', 'wall_a', 'wall_b')
FLUIDS, WALLS = (0, 1), (2, 3)
RHO0, C0 = 1000.0, 15.0
PARAMS = dict(c0=C0, rho0=RHO0, alpha=0.3, nu=0.02, edac_nu=0.05, gx=0.7, gy=-9.81, gz=1.3,
              tdamp=1.0)
EPS_XSPH = 0.4
WALL_ACC = (0.9, -2.5, 0.6)             # wall_b's prescribed acceleration
SENTINEL = 123.0                        # no pass writes this value
FLUID_TVF = ['V', 'rho', 'pavg', 'au', 'av', 'aw', 'auhat', 'avhat', 'awhat', 'ap']
FLUID_EXT = ['V', 'rho', 'au', 'av', 'aw', 'ap', 'ax', 'ay', 'az']
WALL = ['V', 'p', 'wij', 'uf', 'vf', 'wf', 'ug', 'vg', 'wg']
NGHOST = 30
# variant -> (walls, external flow, bql, clamp_p, damped)
VARIANTS = {'internal_bql_damped': (False, False, True, False, True),
            'internal': (False, False, False, False, False),
            'walls_bql': (True, False, True, False, False),
            'walls_damped': (True, False, False, False, True),
            'ext': (True, True, False, False, False),
            'ext_clamp_damped': (True, True, False, True, True)}


@pytest.fixture(autouse=True)
def _cuda_library(gpu_device):
    """these tests must reach libb200sph.so, not an emulation that another module loaded"""
    from pysph_b200 import _lib
    assert os.path.basename(_lib.load()._name) == 'libb200sph.so', _lib.load()._name


def _case(kname, dim, ext, seed=5):
    """The four arrays; the isolated particle and the coincident pair are fluid_a's, one more
    far particle is a wall_a particle with no neighbour but itself"""
    import pysph_b200 as pb
    rs = np.random.RandomState(seed)
    dx = 0.1
    h0 = 1.3 * dx
    k = orc.load().orc_kernel_radius_scale(orc.K_IDS[kname])
    radius = k * 1.2 * h0
    g, pair = _positions(dim, radius, rs, dx, nside={1: 300, 2: 20, 3: 8}[dim])
    lone = g[0] + 3 * radius                # the wall particle with no fluid neighbour
    g = np.concatenate([g, lone[None]])
    n = len(g)
    h = _fix_h(g, h0 * (1 + 0.2 * rs.uniform(-1, 1, n)), k, rs)
    label = rs.randint(0, len(NAMES), n)
    label[[0, pair[0], pair[1]]] = 0
    label[-1] = 2
    vel = [rs.normal(size=n) if d < dim else np.zeros(n) for d in range(3)]
    fluid = pb.get_particle_array_edac_ext if ext else pb.get_particle_array_edac
    pas = []
    for a, name in enumerate(NAMES):
        sel = np.flatnonzero(label == a)
        nk = len(sel)
        props = dict(x=g[sel, 0], y=g[sel, 1] if dim > 1 else np.zeros(nk),
                     z=g[sel, 2] if dim > 2 else np.zeros(nk), h=h[sel],
                     m=RHO0 * dx ** dim * (1 + 0.1 * rs.uniform(-1, 1, nk)),
                     rho=RHO0 * (1 + 0.05 * rs.uniform(-1, 1, nk)),
                     u=vel[0][sel], v=vel[1][sel], w=vel[2][sel])
        if a in FLUIDS:
            pa = fluid(name=name, p=RHO0 * C0 ** 2 * 0.05 * rs.uniform(-1, 1, nk), **props)
            if not ext:
                for d, key in enumerate(('uhat', 'vhat', 'what')):
                    pa.properties[key][:] = props['uvw'[d]] + 0.1 * rs.normal(size=nk) * (d < dim)
            for f in (FLUID_EXT if ext else FLUID_TVF):
                pa.properties[f][:] = SENTINEL
        else:
            pa = pb.get_particle_array_edac_wall(name=name, **props)
            if a == WALLS[1]:
                for key, acc in zip(('au', 'av', 'aw'), WALL_ACC):
                    pa.properties[key][:] = acc
            for f in WALL:
                pa.properties[f][:] = SENTINEL
        if a == 0:
            pa.set_num_real_particles(nk - NGHOST)
        pas.append(pa)
    return pas


def copy_arrays(pas):
    from pysph_b200.particle_array import ParticleArray
    out = []
    for pa in pas:
        q = ParticleArray(name=pa.name, **dict((k, v.copy()) for k, v in pa.properties.items()))
        q.set_num_real_particles(pa.num_real_particles)
        out.append(q)
    return out


def _params(variant):
    walls, ext, bql, clamp, damped = VARIANTS[variant]
    p = dict(PARAMS, pb=0.0 if ext else RHO0 * C0 ** 2, solids=list(WALLS) if walls else [],
             t=0.4 if damped else 1.5)
    return p, walls, ext, bql, clamp


def device_pass(be, variant):
    from pysph_b200 import _lib
    p, walls, ext, bql, clamp = _params(variant)
    prog = _lib.TvfProgram()
    prog.fluid_mask = sum(1 << a for a in FLUIDS)
    prog.solid_mask = sum(1 << a for a in WALLS) if walls else 0
    prog.eqbits = orc.edac_eqbits(p)
    # the average pressure is in group 1 without walls, a Group of its own behind the wall
    # pressure with them (program.py)
    prog.bql = int(bql and not walls)
    prog.passes = 3 | (4 if bql and walls else 0)
    prog.clamp_p = int(clamp)
    prog.eps_xsph = EPS_XSPH if ext else 0.0
    for k in ('pb', 'nu', 'edac_nu', 'c0', 'rho0', 'alpha', 'gx', 'gy', 'gz', 'tdamp', 't'):
        setattr(prog, k, p[k])
    pairs = C.c_int64()
    be.ctx.call('b200sph_tvf_pass', C.byref(prog), C.byref(pairs))
    be.pull_all()
    return pairs.value


def oracle_pass(opas, kname, dim, variant):
    """the oracle's passes in the order of EDACOracleSolver.evaluate"""
    p, walls, ext, bql, clamp = _params(variant)
    o = orc.Oracle(opas, dim, kname)
    o.update_domain()
    o.nnps_update()
    P = o.tvf_program(FLUIDS, orc.edac_eqbits(p), bql=bql and not walls, pb=p['pb'], nu=p['nu'],
                      edac_nu=p['edac_nu'], c0=p['c0'], rho0=p['rho0'], alpha=p['alpha'],
                      gx=p['gx'], gy=p['gy'], gz=p['gz'], tdamp=p['tdamp'], t=p['t'],
                      solids=p['solids'], eps_xsph=EPS_XSPH if ext else 0.0, clamp_p=clamp)
    pairs = o.tvf_pass1(P)
    if walls:
        pairs += o.tvf_wall(P)
        if bql:
            pairs += o.tvf_avgp(P)
    return pairs + o.tvf_pass2(P)


def compare(pas, opas, ext):
    """Every output field untouched (SENTINEL) exactly where the oracle leaves it so; every
    written field within TOL_EVAL of its max |ref| over the array.  Returns the worst error
    per field."""
    worst = {}
    for a, (pa, oa) in enumerate(zip(pas, opas)):
        for f in (WALL if a in WALLS else (FLUID_EXT if ext else FLUID_TVF)):
            got, want = pa.properties[f], oa.properties[f]
            written = want != SENTINEL
            assert np.array_equal(got != SENTINEL, written), (pa.name, f)
            if written.any():
                e = rel_err(got[written], want[written])
                assert e <= TOL_EVAL, (pa.name, f, e)
                worst[f] = max(worst.get(f, 0.0), e)
    return worst


def check_pass(kname, dim, variant):
    import pysph_b200 as pb
    _, walls, ext, bql, clamp = _params(variant)
    pas = _case(kname, dim, ext)
    opas = copy_arrays(pas)
    be = pb.B200Backend(pas)
    pb.B200NNPS(dim, pas, backend=be, kernel=getattr(pb, kname)(dim=dim))
    pairs = device_pass(be, variant)
    assert pairs == oracle_pass(opas, kname, dim, variant) > 0
    worst = compare(pas, opas, ext)
    fa, wa = pas[0], pas[2]
    ng = slice(fa.num_real_particles, None)
    # ghosts: group 1 (real=False) only
    assert np.all(fa.V[ng] != SENTINEL) and np.all(fa.au[ng] == SENTINEL)
    if not ext:
        assert np.all((fa.pavg[ng] != SENTINEL) == (bql and not walls))
    if walls:
        # the wall particle with no fluid neighbour: wij = 0, p = 0, uf = 0, ug = 2 u
        i = wa.get_number_of_particles() - 1
        assert wa.wij[i] == 0.0 and wa.p[i] == 0.0 and wa.uf[i] == 0.0, (wa.wij[i], wa.p[i])
        assert wa.ug[i] == np.float32(2 * np.float32(wa.u[i]))
        if clamp:
            assert np.all(wa.p >= 0.0) and np.any(opas[2].p[:-1] == 0.0)
    else:
        for a in WALLS:
            for f in WALL:
                assert np.all(pas[a].properties[f] == SENTINEL), (a, f)
    return worst


@pytest.mark.parametrize('variant', sorted(VARIANTS))
@pytest.mark.parametrize('kname,dim', KERNEL_DIMS)
def test_tvf_pass_vs_oracle(gpu_device, kname, dim, variant):
    check_pass(kname, dim, variant)
