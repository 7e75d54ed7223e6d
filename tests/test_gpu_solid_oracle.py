"""k_solid_pass1 / k_solid_pass2 -- elastic dynamics -- and k_stage_solid against the fp64 oracle.

test_gpu_solid.py compares one evaluation with six small reference-generated cases (CubicSpline
and WendlandQuintic 2-D only, one set of array constants, random stresses) and trajectories of
the rings.  Here one b200sph_solid_pass runs, for every (kernel, dim) the kernels are
instantiated for, on four arrays: two elastic arrays with different constants (c0_ref, rho_ref,
G, wdeltap, n; one of them without the artificial-stress correction), one rigid `solids` array
(a source of everything, a destination of nothing) and one array that is neither (ignored).
The geometry is the one of the WCSPH pair-kernel test (a jittered lattice, a double-density
cluster, a sparse corner, a coincident pair, an isolated particle) with h varying by +-20 %,
large enough for several CTAs.  The destinations' stress is built to sit where eigen solvers
break (STATES), and the artificial stress r -- formed in fp64, stored in fp32 -- is held per
state to 1e-6 of that state's max |r|.  Then the two ghost modes of group 1 on one GPU, and
one SolidMechStep round after the pass.  test_solid_oracle_on_cpu.py runs the same checks on
the library emulation.
"""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from helpers import rel_err
from oracle import oracle as orc
from test_gpu_parity import TOL_EVAL
from test_gpu_records32_oracle import KERNEL_DIMS, _positions

pytestmark = pytest.mark.gpu

NAMES = ('solid_a', 'solid_b', 'rigid', 'other')
ELASTIC, RIGID, OTHER = (0, 1), 2, 3
SOURCES = (0, 1, 2)
# the array constants: every one differs between the arrays; solid_b has wdeltap = -1 (the
# default: no artificial-stress kernel correction), solid_a's wdeltap is W(dx) (set in _case)
CONSTS = {'solid_a': dict(c0_ref=40.0, rho_ref=1000.0, G=2.0e5, n=4.0),
          'solid_b': dict(c0_ref=25.0, rho_ref=1200.0, G=6.0e4, wdeltap=-1.0, n=3.0),
          'rigid': dict(c0_ref=30.0, rho_ref=1100.0, G=1.0e5, n=2.0),
          'other': dict(c0_ref=35.0, rho_ref=900.0, G=3.0e4, wdeltap=0.5, n=5.0)}
PROG = dict(eps=0.25, alpha=0.7, beta=1.3, eps_xsph=0.37)
SENTINEL = 123.0                        # no pass writes this value
SYM = ('00', '01', '02', '11', '12', '22')
VG = ['v%d%d' % (i, j) for i in range(3) for j in range(3)]
OUT = ['p', 'arho', 'au', 'av', 'aw', 'ax', 'ay', 'az'] + VG + ['r' + k for k in SYM] + \
    ['as' + k for k in SYM]
GROUP2 = ['arho', 'au', 'av', 'aw', 'ax', 'ay', 'az']
# the stress states of the destinations, on S = s - p I (what eigen_sym3 sees).  A = 1e5 is
# the size of p.  straddle_zero: eigenvalues +-1e-10 A next to -A, the tiny pair rotated in
# its own plane (a general rotation would put rounding of A into them: no solver resolves
# them then); range_1e8: -A with two positive eigenvalues of 2e-8 A and 1e-8 A, rotated
STATES = ('zero', 'iso_tension', 'iso_compression', 'pure_shear', 'diag_distinct',
          'repeated_rotated', 'straddle_zero', 'range_1e8', 'random')
STRESS_A = 1e5
R_TOL = 1e-6                            # r per state, of that state's max |r|


@pytest.fixture(autouse=True)
def _cuda_library(gpu_device):
    """these tests must reach libb200sph.so, not an emulation that another module loaded"""
    from pysph_b200 import _lib
    assert os.path.basename(_lib.load()._name) == 'libb200sph.so', _lib.load()._name


def _rotation(rs, planar):
    if planar:                          # in the xy plane
        t = rs.uniform(0, 2 * np.pi)
        c, s = np.cos(t), np.sin(t)
        return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    q, r = np.linalg.qr(rs.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def stress_state(name, A, rs, planar):
    """(S, its eigenvalues as built) for one stress state; planar: no xz / yz components"""
    Q = _rotation(rs, planar)
    eye = np.eye(3)
    if name == 'zero':
        lam, Q = [0.0, 0.0, 0.0], eye
    elif name == 'iso_tension':
        lam, Q = [A, A, A], eye
    elif name == 'iso_compression':
        lam, Q = [-A, -A, -A], eye
    elif name == 'pure_shear':
        S = np.array([[0.0, A, 0.6 * A], [A, 0.0, -0.3 * A], [0.6 * A, -0.3 * A, 0.0]])
        if planar:
            S[[0, 1, 2, 2], [2, 2, 0, 1]] = 0.0
        return S, np.linalg.eigvalsh(S)
    elif name == 'diag_distinct':
        lam, Q = [A, -0.4 * A, 0.7 * A], eye
    elif name == 'repeated_rotated':      # x and z repeated: a rotation about z mixes x and y
        lam = [0.8 * A, -0.3 * A, 0.8 * A]
    elif name == 'straddle_zero':
        lam, Q = [1e-10 * A, -1e-10 * A, -A], _rotation(rs, True)
    elif name == 'range_1e8':
        lam = [-A, 2e-8 * A, 1e-8 * A]
    else:
        S = rs.normal(scale=A, size=(3, 3))
        S = 0.5 * (S + S.T)
        if planar:
            S[[0, 1, 2, 2], [2, 2, 0, 1]] = 0.0
        return S, np.linalg.eigvalsh(S)
    return Q @ np.diag(lam) @ Q.T, np.array(lam)


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _fix_h(g, h, radius_scale, rs, keep=()):
    """no fp32 knife-edge pairs with varying h: |r - k h_i| >= 1e-5 k h_i for both ends of every
    pair (nudge h where one falls on it)"""
    for _ in range(100):
        near = cKDTree(g).query_pairs(radius_scale * h.max() * (1 + 1e-5), output_type='ndarray')
        r = np.linalg.norm(g[near[:, 0]] - g[near[:, 1]], axis=1)
        bad = np.zeros(len(g), bool)
        for side in (0, 1):
            kh = radius_scale * h[near[:, side]]
            bad[near[np.abs(r - kh) < 1e-5 * kh, side]] = True
        if not bad.any():
            return h
        h[bad] *= 1 + 1e-3 * rs.uniform(-1, 1, int(bad.sum()))
    raise AssertionError('knife-edge pairs left')


def _case(kname, dim, full3x3=False, nghost=0, seed=11):
    """The four arrays (see the module doc) and, per particle of the elastic arrays, the name
    of its stress state.  nghost trailing particles of solid_a are ghosts that carry random
    p, s and r (p and r representable in fp32: the pool holds them in fp32)."""
    import pysph_b200 as pb
    rs = np.random.RandomState(seed)
    dx = 0.1
    h0 = 1.3 * dx
    k = orc.load().orc_kernel_radius_scale(orc.K_IDS[kname])
    g, pair = _positions(dim, k * 1.2 * h0, rs, dx, nside={1: 300, 2: 20, 3: 8}[dim])
    n = len(g)
    h = _fix_h(g, h0 * (1 + 0.2 * rs.uniform(-1, 1, n)), k, rs)
    label = rs.randint(0, len(NAMES), n)
    label[[0, pair[0]]] = 0                 # the isolated particle; r = 0 across two arrays
    label[pair[1]] = 1
    planar = dim < 3 and not full3x3
    vel = [rs.normal(size=n) if d < dim else np.zeros(n) for d in range(3)]
    pas, states = [], []
    for a, name in enumerate(NAMES):
        sel = np.flatnonzero(label == a)
        nk = len(sel)
        c = dict(CONSTS[name])
        if 'wdeltap' not in c:
            c['wdeltap'] = orc.kernel_w(kname, dim, dx, h0) * (1.0 if a == 0 else 0.8)
        rho = c['rho_ref'] * (1 + 0.05 * rs.uniform(-1, 1, nk))
        props = dict(x=g[sel, 0], y=g[sel, 1] if dim > 1 else np.zeros(nk),
                     z=g[sel, 2] if dim > 2 else np.zeros(nk), h=h[sel],
                     m=c['rho_ref'] * dx ** dim * (1 + 0.1 * rs.uniform(-1, 1, nk)), rho=rho,
                     u=vel[0][sel], v=vel[1][sel], w=vel[2][sel],
                     cs=c['c0_ref'] * (1 + 0.1 * rs.uniform(-1, 1, nk)))
        pa = pb.get_particle_array_elastic_dynamics(name=name, constants=c, **props)
        nreal = nk - (nghost if a == 0 else 0)
        pa.set_num_real_particles(nreal)
        st = []
        for i in range(nk):
            if a in ELASTIC and i < nreal:
                st.append(STATES[(i + 3 * a) % len(STATES)])
                A = STRESS_A * rs.uniform(0.5, 2.0)
                S, _ = stress_state(st[-1], A, rs, planar)
                p = c['c0_ref'] * c['c0_ref'] * (rho[i] - c['rho_ref'])
                S = S + p * np.eye(3)
            else:                       # carried: ghosts, the rigid array, the other array
                st.append(None)
                S, _ = stress_state('random', STRESS_A, rs, planar)
            for q, (ia, ib) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
                pa.properties['s' + SYM[q]][i] = S[ia, ib]
        for f in OUT:
            pa.properties[f][:] = SENTINEL
        carried = np.arange(nk) >= nreal if a == 0 else np.full(nk, a == RIGID)
        if carried.any():
            pa.p[carried] = _f32(STRESS_A * rs.uniform(-1, 1, int(carried.sum())))
            for key in SYM:
                pa.properties['r' + key][carried] = _f32(
                    0.1 * rs.uniform(-1, 1, int(carried.sum())))
        pas.append(pa)
        states.append(np.array(st, dtype=object))
    assert all(pa.get_number_of_particles() > 0 for pa in pas)
    assert np.flatnonzero(label == 0)[0] == 0
    return pas, states


def copy_arrays(pas):
    from pysph_b200.particle_array import ParticleArray
    out = []
    for pa in pas:
        q = ParticleArray(name=pa.name, constants=dict((k, np.array(v)) for k, v in
                                                       pa.constants.items()),
                          **dict((k, v.copy()) for k, v in pa.properties.items()))
        q.set_num_real_particles(pa.num_real_particles)
        out.append(q)
    return out


def _backend(pas, kname, dim):
    import pysph_b200 as pb
    be = pb.B200Backend(pas)
    pb.B200NNPS(dim, pas, backend=be, kernel=getattr(pb, kname)(dim=dim))
    return be


def _program(pas, grad3d, passes, ghost_group1=0):
    from pysph_b200 import _lib
    prog = _lib.SolidProgram()
    prog.elastic_mask = sum(1 << a for a in ELASTIC)
    prog.source_mask = sum(1 << a for a in SOURCES)
    prog.grad3d, prog.passes, prog.ghost_group1 = int(grad3d), passes, int(ghost_group1)
    for k, v in PROG.items():
        setattr(prog, k, v)
    for a, pa in enumerate(pas):
        for k in ('c0_ref', 'rho_ref', 'wdeltap', 'n', 'G'):
            getattr(prog, k)[a] = float(pa.constants[k][0])
    return prog


def device_pass(be, pas, grad3d, split=False, ghost_group1=0):
    """passes = 3, or 1 then 2 (split); returns the pairs of both groups"""
    total = 0
    for passes in ((1, 2) if split else (3,)):
        pairs = C.c_int64()
        be.ctx.call('b200sph_solid_pass', C.byref(_program(pas, grad3d, passes, ghost_group1)),
                    C.byref(pairs))
        total += pairs.value
    be.pull_all()
    return total


def _oracle(opas, kname, dim):
    o = orc.Oracle(opas, dim, kname)
    o.update_domain()
    o.nnps_update()
    return o


def oracle_pass(opas, kname, dim, grad3d, groups=(1, 2)):
    o = _oracle(opas, kname, dim)
    P = o.solid_program(ELASTIC, SOURCES, grad3d=grad3d, **PROG)
    pairs = 0
    if 1 in groups:
        pairs += o.solid_group1(P)
    if 2 in groups:
        pairs += o.solid_group2(P)
    return pairs


def compare(pas, opas):
    """Every output field untouched (SENTINEL) exactly where the oracle leaves it so; every
    written field within TOL_EVAL of its max |ref| over the array.  Returns the worst error
    per field family."""
    worst = {}
    for pa, oa in zip(pas, opas):
        for f in OUT:
            got, want = pa.properties[f], oa.properties[f]
            written = want != SENTINEL
            assert np.array_equal(got != SENTINEL, written), (pa.name, f)
            if written.any():
                e = rel_err(got[written], want[written])
                assert e <= TOL_EVAL, (pa.name, f, e)
                fam = f.rstrip('0123456789') or f
                worst[fam] = max(worst.get(fam, 0.0), e)
    return worst


def check_r_by_state(pas, opas, states):
    """r per stress state: within R_TOL of the state's max |r|, exactly 0 where no eigenvalue
    of s - p I is positive"""
    for a in ELASTIC:
        pa, oa, st = pas[a], opas[a], states[a]
        for name in STATES:
            sel = st == name
            if not sel.any():
                continue
            got = np.stack([pa.properties['r' + k][sel] for k in SYM])
            want = np.stack([oa.properties['r' + k][sel] for k in SYM])
            if name in ('zero', 'iso_compression'):
                assert np.all(want == 0.0) and np.all(got == 0.0), (pa.name, name)
                continue
            scale = np.max(np.abs(want))
            assert scale > 0.0, (pa.name, name)
            e = np.max(np.abs(got - want)) / scale
            assert e <= R_TOL, (pa.name, name, e)


def _isolated(pa):
    """the destination whose only neighbour is itself: no velocity gradient, no stress rate
    from it, continuity 0, XSPH of itself only (v_ii = 0)"""
    assert pa.v00[0] == 0.0 and pa.arho[0] == 0.0
    for k, u in (('ax', 'u'), ('ay', 'v'), ('az', 'w')):
        assert pa.properties[k][0] == np.float32(pa.properties[u][0]), k


def check_pass(kname, dim, grad3d, full3x3=False, split=False):
    pas, states = _case(kname, dim, full3x3=full3x3)
    opas = copy_arrays(pas)
    be = _backend(pas, kname, dim)
    pairs = device_pass(be, pas, grad3d, split=split)
    opairs = oracle_pass(opas, kname, dim, grad3d)
    assert pairs == opairs > 0
    worst = compare(pas, opas)
    check_r_by_state(pas, opas, states)
    _isolated(pas[0])
    if not grad3d:
        for f in ('v02', 'v12', 'v20', 'v21', 'v22'):
            for a in ELASTIC:
                assert np.all(pas[a].properties[f] == SENTINEL), (a, f)
    return worst


MATRIX = [(k, d, g3) for k, d in KERNEL_DIMS for g3 in ((0, 1) if d == 3 else (0,))]


@pytest.mark.parametrize('split', [False, True], ids=['passes3', 'passes1then2'])
@pytest.mark.parametrize('kname,dim,grad3d', MATRIX)
def test_solid_pass_vs_oracle(gpu_device, kname, dim, grad3d, split):
    check_pass(kname, dim, grad3d, split=split)


def test_solid_pass_2d_full_stress_vs_oracle(gpu_device):
    """the reference's 2-D scheme carries a full 3x3 stress: s02 / s12 != 0 with
    VelocityGradient2D"""
    check_pass('CubicSpline', 2, 0, full3x3=True)


# ---- ghosts on one GPU ------------------------------------------------------------------------
NGHOST = 40


def check_ghosts(kname, dim, ghost_group1, grad3d=0):
    """ghost_group1 = 0: the ghosts of solid_a are sources of group 2 with the p, s and r they
    carry, and nothing is written to them.  ghost_group1 = 1: group 1 runs on them too -- their
    p, r, stress rate and velocity gradient are the oracle's with every particle real --, and
    group 2 of the real particles takes those values."""
    pas, states = _case(kname, dim, nghost=NGHOST)
    ng = slice(pas[0].num_real_particles, None)
    carried = dict((f, pas[0].properties[f][ng].copy()) for f in ['p'] + ['r' + k for k in SYM])
    opas = copy_arrays(pas)
    be = _backend(pas, kname, dim)
    pairs = device_pass(be, pas, grad3d, ghost_group1=ghost_group1)
    # the pairs are those of the real destinations in either mode
    assert pairs == oracle_pass(copy_arrays(opas), kname, dim, grad3d) > 0
    if ghost_group1:
        # group 1 with every particle real, then group 2 from that state with the ghosts back
        nreal = opas[0].num_real_particles
        opas[0].set_num_real_particles(opas[0].get_number_of_particles())
        oracle_pass(opas, kname, dim, grad3d, groups=(1,))
        every = copy_arrays(opas)
        oracle_pass(every, kname, dim, grad3d, groups=(2,))     # the ghosts' stress rate
        opas[0].set_num_real_particles(nreal)
        oracle_pass(opas, kname, dim, grad3d, groups=(2,))
        for k in SYM:
            opas[0].properties['as' + k][ng] = every[0].properties['as' + k][ng]
    else:
        oracle_pass(opas, kname, dim, grad3d)
    worst = compare(pas, opas)
    check_r_by_state(pas, opas, states)
    for f in GROUP2:                    # ghost destinations get no group-2 output
        assert np.all(pas[0].properties[f][ng] == SENTINEL), f
    if not ghost_group1:
        for f, v in carried.items():
            assert np.array_equal(pas[0].properties[f][ng], v), f
        for f in VG + ['as' + k for k in SYM]:
            assert np.all(pas[0].properties[f][ng] == SENTINEL), f
    return worst


@pytest.mark.parametrize('ghost_group1', [0, 1])
@pytest.mark.parametrize('kname,dim', KERNEL_DIMS)
def test_solid_ghosts_vs_oracle(gpu_device, kname, dim, ghost_group1):
    check_ghosts(kname, dim, ghost_group1)


# ---- SolidMechStep after the pass ---------------------------------------------------------------
STEP_FIELDS = ['x', 'y', 'z', 'u', 'v', 'w', 'rho'] + ['s' + k for k in SYM] + \
    ['x0', 'y0', 'z0', 'u0', 'v0', 'w0', 'rho0'] + ['s' + k + '0' for k in SYM]


def check_stage(kname, dim, arr, devdt, dt=2e-5):
    """one round of b200sph_stage_solid (which = 0, 1, 2) on the state the pass left, against
    orc_stage_solid with the device's accelerations; arr = -1 steps every array (the
    integrator does so only when every array has a SolidMechStep), arr = 0 solid_a alone.
    Ghosts never move."""
    pas, _ = _case(kname, dim, nghost=NGHOST)
    be = _backend(pas, kname, dim)
    device_pass(be, pas, 0)
    opas = copy_arrays(pas)             # the device's state, accelerations included
    o = _oracle(opas, kname, dim)
    before = copy_arrays(pas)
    if devdt:
        be.ctx.call('b200sph_time_set', 0.0, dt)
    for which in (0, 1, 2):
        if devdt and which:
            be.ctx.call('b200sph_stage_solid_dev', arr, which)
        else:
            be.ctx.call('b200sph_stage_solid', arr, which, dt)
        for a in (range(len(pas)) if arr < 0 else (arr,)):
            o.stage_solid(a, which, dt)
        be.pull_all()
        for pa, oa, pb_ in zip(pas, opas, before):
            nr = pa.num_real_particles
            for f in STEP_FIELDS:
                got, want = pa.properties[f], oa.properties[f]
                assert np.array_equal(got[nr:], pb_.properties[f][nr:]), (pa.name, f, 'ghost')
                assert rel_err(got, want) <= 1e-13, (which, pa.name, f, rel_err(got, want))
            if arr >= 0 and pa.name != NAMES[arr]:
                for f in STEP_FIELDS:
                    assert np.array_equal(pa.properties[f], pb_.properties[f]), (pa.name, f)
    assert np.any(pas[0].x != before[0].x)


@pytest.mark.parametrize('devdt', [False, True], ids=['dt', 'dev'])
@pytest.mark.parametrize('arr', [-1, 0])
def test_solid_stage_vs_oracle(gpu_device, arr, devdt):
    check_stage('CubicSpline', 3, arr, devdt)
