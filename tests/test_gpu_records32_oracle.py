"""k_pair_list_r32 -- the WCSPH pair kernel on the 32-byte records -- against the fp64 oracle.

The other tests of the 32-byte records compare them with the 48-byte ones on a CubicSpline 3-D
dam break.  Here one pair pass runs, for every (kernel, dim) the kernel is instantiated for, on
six arrays with a Group whose equations depend on the (destination, source) pair, with
parameters unlike the dam break's (beta != 0, eps_xsph != 0.5, the Group's c0 != the EOS c0,
gravity along every axis, a pressure offset p0), and at the edges of its arithmetic:
densities +-25 % around rho0 (clamped in the HG-corrected arrays), two particles at the same
position (r = 0), a destination with no neighbour but itself, and a dense cluster next to a
sparse region (lists of very different length in one warp).  The same case with
B200SPH_RECORDS=48 pins the 48-byte records to the same reference.

Then: EPEC trajectories through the 32-byte records with kernels other than CubicSpline, and
the choice of layout (records32 in b200sph.cu) against the oracle.  Every test here runs on the
GPU; test_records32_oracle_on_cpu.py runs the same checks on the library emulation.
"""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from helpers import ACC_FIELDS, copy_arrays, rel_err
from oracle import oracle as orc
from test_gpu_parity import TOL_EVAL, _compare_state, make_solver, scheme_params

pytestmark = pytest.mark.gpu

# every (kernel, dim) of with_kernel_dim (b200sph.cu)
KERNEL_DIMS = [('CubicSpline', 1), ('CubicSpline', 2), ('CubicSpline', 3),
               ('WendlandQuintic', 2), ('WendlandQuintic', 3),
               ('QuinticSpline', 1), ('QuinticSpline', 2), ('QuinticSpline', 3),
               ('Gaussian', 1), ('Gaussian', 2), ('Gaussian', 3)]
NAMES = ('fluid', 'fluid2', 'wall', 'obstacle', 'wall2', 'probe')
RHO0, C0 = 1000.0, 25.0                 # the EOS of every array
# the Group's parameters: none of them is the dam break's
PROG = dict(c0=30.0, alpha=0.3, beta=0.7, eps_xsph=0.37, gx=0.5, gy=-9.81, gz=1.25)
P0 = 5000.0
SENTINEL = 123.0                        # no pass writes this value
ISOLATED = 0                            # index of the isolated destination in array 0


@pytest.fixture(autouse=True)
def _cuda_library(gpu_device):
    """these tests must reach libb200sph.so, not an emulation that another module loaded"""
    from pysph_b200 import _lib
    assert os.path.basename(_lib.load()._name) == 'libb200sph.so', _lib.load()._name


def _equations():
    """(destination type, source type) -> equation bits"""
    from pysph_b200 import _lib
    CONT, MOM, XSPH = _lib.EQ_CONTINUITY, _lib.EQ_MOMENTUM, _lib.EQ_XSPH
    return {(0, 0): CONT | MOM | XSPH, (0, 5): MOM, (0, 3): CONT | XSPH, (1, 4): MOM | XSPH,
            (2, 0): CONT, (3, 1): XSPH, (4, 2): MOM, (5, 5): CONT | MOM | XSPH}


def _eos_calls(variant):
    """per array (hg, rho0, c0, gamma, p0): 'hg' -- p0 = 0 and three TaitEOSHGCorrection
    arrays; 'p0' -- a plain TaitEOS with the same offset p0 != 0 for every array"""
    if variant == 'hg':
        return [(hg, RHO0, C0, 7.0, 0.0) for hg in (0, 0, 1, 1, 1, 0)]
    return [(0, RHO0, C0, 7.0, P0)] * len(NAMES)


def _positions(dim, radius, rs, dx, nside=None):
    """A jittered lattice (nside particles a side) with a cluster at twice the density in one
    corner, a sparse region in the opposite corner, two particles at the same position and
    one (the first) far from all others.  Returns (positions, indices of the coincident pair)."""
    nside = nside or {1: 60, 2: 16, 3: 8}[dim]
    g = np.mgrid[tuple(slice(0, nside) for _ in range(dim))].reshape(dim, -1).T * dx
    corner = np.all(g < 4 * dx, axis=1)
    sparse = np.all(g >= (nside - 4) * dx, axis=1) & (rs.uniform(size=len(g)) < 0.7)
    g = np.concatenate([g[~sparse], g[corner] + 0.5 * dx])
    g = g + 0.2 * dx * rs.uniform(-1, 1, g.shape)
    far = np.full((1, dim), (nside + 2) * dx + 2 * radius)
    g = np.concatenate([far, g])
    pair = (len(g) // 2, len(g) // 2 + 1)
    g[pair[1]] = g[pair[0]]
    # no fp32 knife-edge pairs: |r - k h| >= 1e-5 h for every pair, in fp64 (nudge a particle
    # off the edge where one falls on it)
    keep = {0, pair[0], pair[1]}
    for _ in range(50):
        near = cKDTree(g).query_pairs(radius * (1 + 1e-5), output_type='ndarray')
        r = np.linalg.norm(g[near[:, 0]] - g[near[:, 1]], axis=1)
        edge = near[r > radius * (1 - 1e-5)]
        if not len(edge):
            break
        for i, j in edge:
            k = j if j not in keep else i
            g[k] += 1e-3 * dx * rs.uniform(-1, 1, dim)
    near = cKDTree(g).query_pairs(radius * (1 + 1e-5), output_type='ndarray')
    r = np.linalg.norm(g[near[:, 0]] - g[near[:, 1]], axis=1)
    assert np.all(r <= radius * (1 - 1e-5)), 'a pair at |r - k h| < 1e-5 h'
    assert np.all(np.linalg.norm(g[1:] - g[0], axis=1) > 1.5 * radius)
    return g, pair


def _case(kname, dim, seed=7):
    """Six arrays (types 0-5) of one jittered lattice, every particle labelled at random
    (every (destination, source) pair of types occurs), uniform h = 1.3 dx and m, densities
    +-25 % around rho0, random velocities."""
    import pysph_b200 as pb
    rs = np.random.RandomState(seed)
    dx = 0.1
    h = 1.3 * dx
    kernel = getattr(pb, kname)(dim=dim)
    g, pair = _positions(dim, kernel.radius_scale * h, rs, dx)
    n = len(g)
    label = rs.randint(0, len(NAMES), n)
    label[[0, pair[0], pair[1]]] = 0         # momentum, continuity and XSPH from type 0
    rho = RHO0 * (1 + 0.25 * rs.uniform(-1, 1, n))
    vel = [rs.normal(size=n) if d < dim else np.zeros(n) for d in range(3)]
    pas = []
    for k, name in enumerate(NAMES):
        sel = label == k
        nk = int(sel.sum())
        xyz = [g[sel, d] if d < dim else np.zeros(nk) for d in range(3)]
        pas.append(pb.get_particle_array_wcsph(
            name=name, x=xyz[0], y=xyz[1], z=xyz[2], h=np.full(nk, h),
            m=np.full(nk, RHO0 * dx ** dim), rho=rho[sel], u=vel[0][sel], v=vel[1][sel],
            w=vel[2][sel]))
    assert all(pa.get_number_of_particles() > 0 for pa in pas)
    assert np.flatnonzero(label == 0)[ISOLATED] == 0
    params = dict(fluids=list(NAMES[:2]), solids=list(NAMES[2:]), dim=dim, rho0=RHO0, c0=C0,
                  h0=h, hdx=1.3, gamma=7.0, alpha=0.25, beta=0.0, hg_correction=True,
                  tensile_correction=False, dt0=1e-4, cfl=0.3, integrator='EPEC')
    return pas, params


def _solver(monkeypatch, kname, dim, records, pas, params):
    """The solver, initialised: TaitEOSHGCorrection has clamped the solids' rho in the pool,
    so the state the oracle starts from is pulled after this"""
    import pysph_b200 as pb
    if records == '48':
        monkeypatch.setenv('B200SPH_RECORDS', '48')
    else:
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    s = pb.make_wcsph_solver(pas, dict(params), getattr(pb, kname)(dim=dim))
    s.initialise()
    s.pull()
    return s


def _device_pass(s, pas, eqs, eos, prog_kw, tensile=False, nu=0.0):
    """One b200sph_pair_pass after the given b200sph_eos calls (None: no call for that
    array), every acceleration field at SENTINEL before it.  Returns (pairs, r32 launches)."""
    from pysph_b200 import _lib
    be = s.backend
    n0 = be.stats()['pair_launches_r32']
    prog = _lib.PairProgram()
    for (d, src), bits in eqs.items():
        prog.eqmask[d][src] = bits
    for k, v in prog_kw.items():
        setattr(prog, k, v)
    prog.tensile_correction = int(tensile)
    prog.nu, prog.eta = nu, 0.01
    for a, call in enumerate(eos):
        if call is not None:
            be.ctx.call('b200sph_eos', a, *call, 0)
    for a, pa in enumerate(pas):
        for k in ACC_FIELDS:
            pa.properties[k][:] = SENTINEL
        be.push_real_array(a, ACC_FIELDS)
    pairs = C.c_int64()
    be.ctx.call('b200sph_pair_pass', C.byref(prog), C.byref(pairs))
    s.pull()
    return pairs.value, be.stats()['pair_launches_r32'] - n0


def _oracle_pass(opas, kname, dim, eqs, eos, prog_kw, tensile=False, nu=0.0):
    bit = _oracle_bits()
    for pa in opas:
        for k in ACC_FIELDS:
            pa.properties[k][:] = SENTINEL
    o = orc.Oracle(opas, dim, kname)
    o.update_domain()
    o.nnps_update()
    for a, call in enumerate(eos):
        if call is not None:
            o.eos(a, *call)
    oeqs = [(o_bit, d, [src]) for (d, src), bits in sorted(eqs.items())
            for b, o_bit in bit.items() if bits & b]
    return o.pair_pass(oeqs, real_only=True, tensile_correction=tensile, nu=nu, eta=0.01,
                       **prog_kw)


def _oracle_bits():
    from pysph_b200 import _lib
    return {_lib.EQ_CONTINUITY: orc.EQ_CONT, _lib.EQ_MOMENTUM: orc.EQ_MOM,
            _lib.EQ_XSPH: orc.EQ_XSPH, _lib.EQ_LAMINAR: orc.EQ_LAMINAR}


def _compare(pas, opas):
    """Every field untouched (SENTINEL) exactly where the oracle leaves it so, every written
    field within TOL_EVAL of its max |ref|.  Returns the worst error."""
    worst = 0.0
    for pa, oa in zip(pas, opas):
        for k in ACC_FIELDS:
            got, want = pa.properties[k], oa.properties[k]
            written = want != SENTINEL
            assert np.array_equal(got != SENTINEL, written), (pa.name, k)
            if written.any():
                e = rel_err(got[written], want[written])
                assert e <= TOL_EVAL, (pa.name, k, e)
                worst = max(worst, e)
    return worst


def _check_isolated(pa, vel):
    """the destination whose only neighbour is itself: no cfl pair (dt_cfl = 0), gravity
    only, XSPH of itself (v_ii = 0), continuity 0"""
    i = ISOLATED
    assert pa.dt_cfl[i] == 0.0
    for k, g in (('au', 'gx'), ('av', 'gy'), ('aw', 'gz')):
        assert pa.properties[k][i] == np.float32(PROG[g]), k
    for k, u in zip(('ax', 'ay', 'az'), vel):
        assert pa.properties[k][i] == np.float32(u), k
    assert pa.arho[i] == 0.0


def check_pass_vs_oracle(monkeypatch, kname, dim, variant, records):
    pas, params = _case(kname, dim)
    s = _solver(monkeypatch, kname, dim, records, pas, params)
    opas = copy_arrays(pas)
    vel = [pas[0].properties[k][ISOLATED] for k in ('u', 'v', 'w')]
    eqs, eos = _equations(), _eos_calls(variant)
    pairs, r32 = _device_pass(s, pas, eqs, eos, PROG)
    opairs = _oracle_pass(opas, kname, dim, eqs, eos, PROG)
    assert r32 == (1 if records == '32' else 0)
    assert pairs == opairs > 0
    worst = _compare(pas, opas)
    _check_isolated(pas[0], vel)
    return worst


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('variant', ['hg', 'p0'])
@pytest.mark.parametrize('kname,dim', KERNEL_DIMS)
def test_pair_pass_vs_oracle(gpu_device, monkeypatch, kname, dim, variant, records):
    check_pass_vs_oracle(monkeypatch, kname, dim, variant, records)


# ---- trajectories through the 32-byte records with kernels other than CubicSpline ----------
def _dam_break(kname, vscale=2.0, seed=5):
    """The 2-D dam break (WendlandQuintic) with h kept fixed, or a small 3-D one (QuinticSpline:
    radius 3 h, more list entries per destination); random fluid velocities use up the list
    skin within the run"""
    from pysph_b200 import geometry as geo
    if kname == 'WendlandQuintic':
        pas = geo.dam_break_2d_particles(dx=0.03)
        params = dict(geo.dam_break_2d_params(dx=0.03), update_h=False, integrator='EPEC')
    else:
        pas = geo.dam_break_3d_particles(dx=0.08)
        params = geo.dam_break_3d_params(0.08)
    rs = np.random.RandomState(seed)
    f = pas[0]
    for k in ('u', 'v', 'w')[:params['dim']]:
        f.properties[k][:] = rs.normal(scale=vscale, size=f.x.size)
    return pas, params


def check_trajectory(kname, steps=20):
    pas, params = _dam_break(kname)
    opas = copy_arrays(pas)
    s = make_solver(pas, scheme_params(params), kname)
    o = orc.WCSPHOracleSolver(opas, params, kname, threads=4)
    s.a_eval.count_pairs = True
    s.initialise()
    o.initialise()
    assert s.a_eval.last_pairs == o.pairs_last_eval
    s.a_eval.count_pairs = False
    for _ in range(steps):
        s.step()
        o.step()
    s.pull()
    st = s.backend.stats()
    assert st['pair_launches_r32'] == st['pair_launches'] > 0, st
    assert st['list_builds'] >= 2, st
    assert abs(s.t - o.t) <= 1e-5 * o.t
    _compare_state(pas, opas, tol_pos=1e-6, tol_vel=1e-6, tol_rho=1e-7,
                   h0=params['h0'], c0=params['c0'], rho0=params['rho0'])


@pytest.mark.parametrize('kname', ['WendlandQuintic', 'QuinticSpline'])
def test_trajectory_vs_oracle(gpu_device, kname):
    check_trajectory(kname)


# ---- the choice of layout (records32 in b200sph.cu) ------------------------------------------
# case -> does the pass take the 32-byte records?
LAYOUT_CASES = {
    'gamma_not_7': False,           # one array with gamma = 6
    'c0_differs': False,            # one array with another c0
    'rho0_differs': False,          # one array with another rho0
    'p0_next_to_hg': False,         # every array p0 != 0: the HG-corrected ones count it as 0
    'tensile': False,
    'laminar': False,               # a LaminarViscosity bit in the Group
    'no_eos_call': False,           # one array without an EOS call in this pass
    'p0_of_hg_ignored': True,       # p0 != 0 on the HG-corrected arrays only: every offset is 0
    'empty_other_eos': True,        # an empty array with gamma = 6 ...
    'empty_no_eos': True,           # ... or without an EOS call: arrays with n == 0 do not count
    'rho0_changes': True,           # rho0 1000, then 1010 on the same context (below)
}


def check_layout(monkeypatch, case, kname='QuinticSpline', dim=2):
    import pysph_b200 as pb
    from pysph_b200 import _lib
    pas, params = _case(kname, dim)
    eqs, eos = _equations(), _eos_calls('hg')
    kw = {}
    if case == 'gamma_not_7':
        eos[3] = (1, RHO0, C0, 6.0, 0.0)
    elif case == 'c0_differs':
        eos[4] = (1, RHO0, 1.1 * C0, 7.0, 0.0)
    elif case == 'rho0_differs':
        eos[1] = (0, 1.005 * RHO0, C0, 7.0, 0.0)
    elif case in ('p0_next_to_hg', 'p0_of_hg_ignored'):
        eos = [(hg, r, c, g, P0 if (hg or case == 'p0_next_to_hg') else 0.0)
               for hg, r, c, g, _ in eos]
    elif case == 'tensile':
        kw['tensile'] = True
    elif case == 'laminar':
        eqs[(0, 0)] |= _lib.EQ_LAMINAR
        kw['nu'] = 0.05
    elif case == 'no_eos_call':
        eos[5] = None
    elif case.startswith('empty'):
        pas.append(pb.get_particle_array_wcsph(name='empty', x=np.zeros(0)))
        params['solids'].append('empty')
        eos.append((0, RHO0, C0, 6.0, 0.0) if case == 'empty_other_eos' else None)
    s = _solver(monkeypatch, kname, dim, '32', pas, params)
    for k in range(2 if case == 'rho0_changes' else 1):
        if k == 1:
            # rho0 and rho x 1.01 (delta stays small).  The push of rho alone makes the next
            # pass repack the records; what this pins is that the repack forms delta with
            # the new rho0 (rec32_rho0), which the kernel's rho0 and Tait constants assume
            eos = [(hg, 1.01 * r, c, g, p0) for hg, r, c, g, p0 in eos]
            for a, pa in enumerate(pas):
                pa.rho[:] *= 1.01
                s.backend.push_real_array(a, ['rho'])
        opas = copy_arrays(pas)
        pairs, r32 = _device_pass(s, pas, eqs, eos, PROG, **kw)
        opairs = _oracle_pass(opas, kname, dim, eqs, eos, PROG, **kw)
        assert r32 == int(LAYOUT_CASES[case])
        assert pairs == opairs > 0
        _compare(pas, opas)


@pytest.mark.parametrize('case', sorted(LAYOUT_CASES))
def test_layout_choice_vs_oracle(gpu_device, monkeypatch, case):
    check_layout(monkeypatch, case)

