"""What the persistent neighbour lists hold, against an fp64 brute force, destination by
destination, while a build is reused up to the limit of its skin.

The lists promise (pair_list.cuh): k_list_build stores every candidate with
r^2 < (k h_i + S)^2 or r^2 < (k h_j + S)^2, and a build stays valid while
2 max|x - x_build| + k max(h - h_build) <= 0.98 S; while it is valid the lists contain every pair
the exact accept test can take.  A pair the lists lose sits at the edge of the support, where W
and grad W are nearly 0, so fields and trajectories barely notice it.  Here a user Equation run
by the generic fallback (codegen.py: it walks the same cnt / lst arrays with the exact accept
test) sums, per destination, the number of sources it accepts, sum key and sum key^2 of a random
integer key below 2^20 on every particle: exact in fp64, and together they name a lost or extra
pair.  The reference is a plain numpy fp64 brute force over all pairs, with the periodic images
materialised.  No candidate lies within 1e-5 k h of either support radius, in any state a test
visits, so the comparison is exact.

The skin is fixed (B200SPH_SKIN=0.1, B200SPH_SKIN_ADAPT=0), so S = 0.1 k hmax is known before
the particles are placed: pairs are put in the skin shell, at k h + f S, and moved towards each
other so that the drift uses up 0.97 S (the lists must be reused) or just over 0.98 S (they must
be rebuilt).  Every move asserts the path it took.  Then the hand-written consumers on the moved
skin-shell state: the pair counts of b200sph_pair_pass on both record layouts (a Group without
wall <- wall equations), of b200sph_tvf_pass (EDAC with solid walls) and of b200sph_solid_pass
(elastic dynamics), each against the brute force over the pairs its passes walk.

Every test here runs on the GPU; test_neighbour_lists_on_cpu.py runs the same checks on the
library emulation.
"""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SKIN = 0.1                  # B200SPH_SKIN: S = SKIN * k * hmax
MARGIN = 0.98               # drift_within_skin
DX = 0.1
HDX = 1.2
RHO0, C0 = 1000.0, 25.0
BAND = 1e-5                 # no candidate within BAND * k h of a support radius
F_SHELL = (0.3, 0.6, 0.9, 0.95)
SIG = ('nb', 'ks', 'kq')    # accepted sources, sum key, sum key^2
SIG2 = ('nb2', 'ks2', 'kq2')


@pytest.fixture(autouse=True)
def _cuda_library(gpu_device):
    """these tests must reach libb200sph.so, not an emulation that another module loaded"""
    from pysph_b200 import _lib
    assert os.path.basename(_lib.load()._name) == 'libb200sph.so', _lib.load()._name


_EQS = []


def _signature_equations():
    """two user Equations with the same body on different properties (two Groups can then
    run on overlapping destinations)"""
    if _EQS:
        return _EQS
    import pysph_b200 as pb

    class Signature(pb.Equation):
        def initialize(self, d_idx, d_nb, d_ks, d_kq):
            d_nb[d_idx] = 0.0
            d_ks[d_idx] = 0.0
            d_kq[d_idx] = 0.0

        def loop(self, d_idx, d_nb, d_ks, d_kq, s_idx, s_key):
            d_nb[d_idx] += 1.0
            d_ks[d_idx] += s_key[s_idx]
            d_kq[d_idx] += s_key[s_idx] * s_key[s_idx]

    class Signature2(pb.Equation):
        def initialize(self, d_idx, d_nb2, d_ks2, d_kq2):
            d_nb2[d_idx] = 0.0
            d_ks2[d_idx] = 0.0
            d_kq2[d_idx] = 0.0

        def loop(self, d_idx, d_nb2, d_ks2, d_kq2, s_idx, s_key):
            d_nb2[d_idx] += 1.0
            d_ks2[d_idx] += s_key[s_idx]
            d_kq2[d_idx] += s_key[s_idx] * s_key[s_idx]

    _EQS.extend([(Signature, SIG), (Signature2, SIG2)])
    return _EQS


# ---- the reference ----------------------------------------------------------------------------
def _images(box):
    """the image shifts: -L, 0, +L along every periodic axis (a periodic axis is at least
    k hmax + S long, so no pair is accepted across two periods)"""
    if box is None:
        return [np.zeros(3)]
    lo, hi, per = box
    axes = [(-1, 0, 1) if per[d] else (0,) for d in range(3)]
    return [np.array(c, dtype=float) * (np.asarray(hi) - np.asarray(lo))
            for c in itertools.product(*axes)]


def brute_force(X, H, key, owner, narr, kr, box=None, chunk=256):
    """fp64, all pairs and images: per particle i and source array s the number of sources j of
    s with r^2 < (k h_i)^2 or r^2 < (k h_j)^2, sum key_j and sum key_j^2 (int64, exact); and the
    pairs (i, j) with a distance within BAND k h of k h_i or k h_j"""
    n = len(X)
    R = kr * H
    cnt = np.zeros((n, narr), dtype=np.int64)
    ks = np.zeros((n, narr), dtype=np.int64)
    kq = np.zeros((n, narr), dtype=np.int64)
    band = []
    onehot = np.zeros((n, narr), dtype=np.int64)
    onehot[np.arange(n), owner] = 1
    kk = onehot * key[:, None]
    kk2 = onehot * (key * key)[:, None]
    for sh in _images(box):
        Y = X + sh
        for a in range(0, n, chunk):
            b = min(n, a + chunk)
            d = X[a:b, None, :] - Y[None, :, :]
            r2 = np.einsum('ijk,ijk->ij', d, d)
            acc = (r2 < (R[a:b, None] ** 2)) | (r2 < (R[None, :] ** 2))
            A = acc.astype(np.int64)
            cnt[a:b] += A @ onehot
            ks[a:b] += A @ kk
            kq[a:b] += A @ kk2
            r = np.sqrt(r2)
            bad = (np.abs(r - R[a:b, None]) < BAND * R[a:b, None]) | \
                  (np.abs(r - R[None, :]) < BAND * R[None, :])
            for i, j in zip(*np.nonzero(bad)):
                band.append((a + i, j))
    return cnt, ks, kq, band


# ---- the harness ------------------------------------------------------------------------------
class Lists(object):
    """Particle arrays with a random integer key, one generic Group per entry of `groups`
    ((Signature class index, [(dest, sources), ...])), a B200NNPS on a fixed skin.  `moving`:
    per array, a mask of the particles the test will move or whose h it will change (the others
    are nudged first when a pair falls on a knife edge); `keep`: the particles never nudged."""

    def __init__(self, monkeypatch, dim, arrays, groups, box=None, zorder=0, records=None,
                 kname='CubicSpline', seed=11, moving=None, keep=None, extra_states=()):
        import pysph_b200 as pb
        monkeypatch.setenv('B200SPH_SKIN', repr(SKIN))
        monkeypatch.setenv('B200SPH_SKIN_ADAPT', '0')
        monkeypatch.setenv('B200SPH_ZORDER', str(int(zorder)))
        if records:
            monkeypatch.setenv('B200SPH_RECORDS', records)
        else:
            monkeypatch.delenv('B200SPH_RECORDS', raising=False)
        self.dim, self.box = dim, box
        self.rs = np.random.RandomState(seed)
        self.names = [a[0] for a in arrays]
        self.X = np.concatenate([np.asarray(a[1], dtype=float) for a in arrays])
        self.H = np.concatenate([np.asarray(a[2], dtype=float) for a in arrays])
        self.owner = np.concatenate([np.full(len(a[1]), k) for k, a in enumerate(arrays)])
        self.start = np.concatenate([[0], np.cumsum([len(a[1]) for a in arrays])])
        self.key = self.rs.randint(0, 1 << 20, len(self.X)).astype(np.int64)
        self.moving = np.zeros(len(self.X), dtype=bool) if moving is None else \
            np.concatenate([np.asarray(m, dtype=bool) for m in moving])
        self.keep = np.zeros(len(self.X), dtype=bool) if keep is None else \
            np.concatenate([np.asarray(m, dtype=bool) for m in keep])
        self.kernel = getattr(pb, kname)(dim=dim)
        self.kr = self.kernel.radius_scale
        # the states the test will visit, as (dX, dH) from the initial one: no knife edge in any
        self._clear_band([(0.0, 0.0)] + list(extra_states))
        eqs = _signature_equations()
        self.groups = [(eqs[c][1], spec) for c, spec in groups]
        self.pas = []
        for k, name in enumerate(self.names):
            sl = slice(self.start[k], self.start[k + 1])
            xyz = self.X[sl]
            pa = pb.get_particle_array_wcsph(
                name=name, x=xyz[:, 0].copy(), y=xyz[:, 1].copy(), z=xyz[:, 2].copy(),
                h=self.H[sl].copy(), m=np.full(len(xyz), RHO0 * DX ** dim),
                rho=np.full(len(xyz), RHO0))
            for p in ('key',) + SIG + SIG2:
                pa.add_property(p)
            pa.properties['key'][:] = self.key[sl]
            self.pas.append(pa)
        self.ae = pb.B200AccelerationEval(
            self.pas, [pb.Group(equations=[eqs[c][0](dest=d, sources=list(s)) for d, s in spec])
                       for c, spec in groups], self.kernel)
        self.be = self.ae.backend
        domain = None
        if box is not None:
            lo, hi, per = box
            domain = pb.DomainManager(
                xmin=lo[0], xmax=hi[0], ymin=lo[1], ymax=hi[1], zmin=lo[2], zmax=hi[2],
                periodic_in_x=bool(per[0]), periodic_in_y=bool(per[1]),
                periodic_in_z=bool(per[2]))
        self.nn = pb.B200NNPS(dim, self.pas, backend=self.be, kernel=self.kernel, domain=domain)
        self.ae.set_nnps(self.nn)
        self.S = SKIN * self.kr * self.H.max()
        need, S = self.drift()
        assert S == pytest.approx(self.S, rel=1e-12, abs=0.0), (S, self.S)

    # -- knife edges -------------------------------------------------------------------------
    def _band(self, X, H):
        return brute_force(X, H, self.key, self.owner, len(self.names), self.kr, self.box)[3]

    def _clear_band(self, states):
        """nudge particles the test does not move until no pair of any planned state is within
        BAND k h of a support radius"""
        for _ in range(60):
            bad = set()
            for dX, dH in states:
                bad.update(self._band(self.X + dX, self.H + dH))
            if not bad:
                return
            for i, j in sorted(bad):
                # never a kept particle; a static one before one the test moves
                k = min((i, j), key=lambda q: (bool(self.keep[q]), bool(self.moving[q])))
                assert not self.keep[k], 'a knife-edge pair of two kept particles'
                # a particle the test moves is nudged less: it shifts all its states alike, and
                # its distance to a partner in the skin shell by far less than the f steps
                step = 2e-4 * DX if self.moving[k] else 1e-3 * DX
                self.X[k, :self.dim] += step * self.rs.uniform(-1, 1, self.dim)
        raise AssertionError('could not clear the knife-edge band')

    # -- the library ---------------------------------------------------------------------------
    def drift(self):
        out = (C.c_double * 2)()
        self.be.ctx.call('b200sph_nnps_drift', out)
        return out[0], out[1]

    def stats(self):
        return self.be.stats()

    def _push(self, h=False):
        for k, pa in enumerate(self.pas):
            sl = slice(self.start[k], self.start[k + 1])
            pa.x[:], pa.y[:], pa.z[:] = self.X[sl, 0], self.X[sl, 1], self.X[sl, 2]
            props = ['x', 'y', 'z']
            if h:
                pa.h[:] = self.H[sl]
                props.append('h')
            self.be.push(k, props)

    def signature(self, props=SIG):
        """one evaluation; per array the device's (count, sum key, sum key^2), as int64"""
        self.ae.compute(0.0, 0.0)
        self.be.pull_all(list(props))
        out = []
        for pa in self.pas:
            v = [pa.properties[p] for p in props]
            for a in v:
                assert np.all(a == np.round(a)), 'a signature that is not an integer'
            out.append([a.astype(np.int64) for a in v])
        return out

    def optimistic_pass(self):
        """the evaluation between update(deferred=True) and confirm(): a pair pass (continuity
        for the Groups' pairs).  A generic Group is not one: its launch refuses to run on a
        deferred check that failed and was never confirmed."""
        from pysph_b200 import _lib
        prog = _lib.PairProgram()
        for _, spec in self.groups:
            for d, sources in spec:
                for s in sources:
                    prog.eqmask[self.names.index(d)][self.names.index(s)] = _lib.EQ_CONTINUITY
        self.be.ctx.call('b200sph_pair_pass', C.byref(prog), None)

    def reference(self):
        return brute_force(self.X, self.H, self.key, self.owner, len(self.names), self.kr,
                           self.box)

    def check(self):
        """the signature of every Group equals the brute force's, destination by destination;
        returns the reference's pair count of every Group"""
        ref = self.reference()
        assert not ref[3], 'a knife-edge pair %s' % (ref[3][:4],)
        pairs = []
        for props, spec in self.groups:
            got = self.signature(props)
            n_pairs = 0
            for dest, sources in spec:
                d = self.names.index(dest)
                cols = [self.names.index(s) for s in sources]
                sl = slice(self.start[d], self.start[d + 1])
                want = [r[sl][:, cols].sum(axis=1) for r in ref[:3]]
                n_pairs += int(want[0].sum())
                for p, g, w in zip(props, got[d], want):
                    bad = np.flatnonzero(g != w)
                    assert not len(bad), self._explain(dest, sources, p, bad, g, w)
            pairs.append(n_pairs)
        return pairs

    def _explain(self, dest, sources, prop, bad, got, want):
        i = int(bad[0])
        g = self.start[self.names.index(dest)] + i
        d = self.X[g] - self.X
        r = np.sqrt(np.einsum('ij,ij->i', d, d))
        near = np.flatnonzero((r < self.kr * (self.H[g] + self.H.max()) + self.S))
        return ('%s of %d destinations of %r <- %s differ; first: %s[%d] = %d, brute force %d '
                '(h %.6g; sources within reach: %s)'
                % (prop, len(bad), dest, sources, prop, i, got[i], want[i], self.H[g],
                   [(self.names[self.owner[j]], int(j - self.start[self.owner[j]]),
                     round(float(r[j] / (self.kr * max(self.H[g], self.H[j]))), 5))
                    for j in near[:40]]))

    def move(self, dX=0.0, dH=0.0, path='reuse', need=None, deferred=False):
        """apply the move, assert the drift the library measures and the path the update takes
        (reuse: one light update; rebuild: one full build; with deferred=True the rebuild is
        found by confirm() after an evaluation on the stale lists), then the signatures"""
        self.X = self.X + dX
        h = np.any(dH != 0.0)
        self.H = self.H + dH
        self._push(h)
        got_need, S = self.drift()
        assert S == pytest.approx(self.S, rel=1e-12, abs=0.0)
        if need is not None:
            assert abs(got_need - need) <= 2e-3 * S, (got_need / S, need / S)
        assert (got_need <= MARGIN * S) == (path == 'reuse'), (got_need / S, path)
        st0 = self.stats()
        self.nn.update(deferred=deferred)
        st1 = self.stats()
        if path == 'reuse':
            assert (st1['light_updates'] - st0['light_updates'],
                    st1['full_builds'] - st0['full_builds']) == (1, 0)
            if deferred:
                self.optimistic_pass()
                assert self.nn.confirm() is False
        elif deferred:
            # optimistic: the update reuses the lists, the evaluation runs on them, confirm()
            # then asks for the repeat
            assert st1['full_builds'] == st0['full_builds']
            self.optimistic_pass()
            assert self.nn.confirm() is True
            st2 = self.stats()
            assert st2['deferred_failed'] == st0['deferred_failed'] + 1
            assert st2['light_updates'] == st0['light_updates']
            self.nn.update()
            st1 = self.stats()
            assert st1['full_builds'] - st0['full_builds'] == 1
        else:
            assert (st1['light_updates'] - st0['light_updates'],
                    st1['full_builds'] - st0['full_builds']) == (0, 1)
        if path != 'reuse':
            # a new build: S from the current hmax, nothing used up yet
            self.S = SKIN * self.kr * self.H.max()
            need0, S = self.drift()
            assert S == pytest.approx(self.S, rel=1e-12, abs=0.0)
        return self.check()


# ---- geometry ---------------------------------------------------------------------------------
NSIDE = {1: 30, 2: 20, 3: 16}


def _lattice(dim, nside, rs, dx=DX, jitter=0.2):
    g = np.mgrid[tuple(slice(0, nside) for _ in range(dim))].reshape(dim, -1).T * dx
    g = g + jitter * dx * rs.uniform(-1, 1, g.shape)
    return np.concatenate([g, np.zeros((len(g), 3 - dim))], axis=1)


def _grid(X, kr, hmax):
    """where the pairs are planned: the internal cell grid a non-periodic build of these
    positions should get (the rule of b200sph_nnps_update: bounds padded by 1 %, cell edge
    k hmax + S) -- origin, edge, cells.  What the library really built is read back by
    _assert_crossings."""
    mn, mx = X.min(axis=0), X.max(axis=0)
    ln = mx - mn
    mn, mx = mn - 0.01 * ln, mx + 0.01 * ln
    cell = kr * hmax * (1.0 + SKIN)
    nc = np.maximum(np.ceil((mx - mn) / cell).astype(int), 1)
    return mn, cell, nc


def _directions(dim):
    return [np.array(e + (0,) * (3 - dim), dtype=float)
            for e in itertools.product((-1, 0, 1), repeat=dim) if any(e)]


def _approach_pairs(dim, static, kr, h, rs, fs=F_SHELL, within=None):
    """pairs at distance k h + f S across every neighbour-cell direction: the midpoint of a pair
    on an interior corner of the cell grid the `static` particles span, the pair along the
    direction (on the axes the direction does not cross, in the middle of the cell), one corner
    per pair, both members inside the box `within` (default: the static particles' bounds).
    Returns (positions [2 n, 3], unit directions [n, 3] from the first to the second member)."""
    mn, cell, nc = _grid(static, kr, h)
    lo, hi = within if within is not None else (static.min(axis=0), static.max(axis=0))
    corners = list(itertools.product(*[range(1, nc[d]) if d < dim else (0,) for d in range(3)]))
    corners = [corners[k] for k in rs.permutation(len(corners))]
    S = SKIN * kr * h
    P, U = [], []
    for e in _directions(dim):
        for f in fs:
            u = e / np.linalg.norm(e)
            r = kr * h + f * S
            for k, c in enumerate(corners):
                mid = mn + np.asarray(c) * cell + np.where(e == 0, 0.5 * cell, 0.0)
                mid[dim:] = 0.0
                p = [mid - 0.5 * r * u, mid + 0.5 * r * u]
                if all(np.all(q[:dim] > lo[:dim]) and np.all(q[:dim] < hi[:dim]) for q in p):
                    break
            else:
                raise AssertionError('no corner left for a pair')
            del corners[k]
            P += p
            U.append(u)
    return np.array(P), np.array(U)


def _assert_crossings(L, first, second):
    """the pairs (L.X[first], L.X[second]) cross every neighbour-cell direction of the grid the
    library built: its origin (b200sph_get_grid's xmin: the padded bounds) and its internal cell
    edge (the reference's cell size k hmax plus the skin S b200sph_nnps_drift reports)"""
    origin = np.asarray(L.nn.xmin)
    cell = L.nn.cell_size + L.drift()[1]
    assert cell == pytest.approx(L.kr * L.H.max() + L.S, rel=1e-12)
    cidx = np.floor((L.X - origin) / cell).astype(int)
    seen = {tuple(d[:L.dim]) for d in cidx[second] - cidx[first]}
    assert seen == {tuple(e.astype(int)[:L.dim]) for e in _directions(L.dim)}, seen


def _toward(U, a):
    """the displacement of every pair member towards its partner by a"""
    return np.stack([a * U, -a * U], axis=1).reshape(-1, 3)


def _shell_case(monkeypatch, dim, zorder, seed=3, records=None, arrays=1, moves=(0.25, 0.485)):
    """jittered lattice (h = 1.2 dx) + approach pairs in the skin shell.  moves: the planned
    cumulative approach of each member, in units of S"""
    rs = np.random.RandomState(seed)
    h = HDX * DX
    kr = 2.0                      # CubicSpline
    lat = _lattice(dim, NSIDE[dim], rs)
    P, U = _approach_pairs(dim, lat, kr, h, rs)
    S = SKIN * kr * h
    X = np.concatenate([lat, P])
    n = len(X)
    moving = np.zeros(n, dtype=bool)
    moving[len(lat):] = True
    states = []
    for a in moves:
        dX = np.zeros((n, 3))
        dX[len(lat):] = _toward(U, a * S)
        states.append((dX, 0.0))
    H = np.full(n, h)
    order = np.arange(n)
    if arrays == 1:
        arr = [('fluid', X, H)]
        mov = [moving]
        groups = [(0, [('fluid', ['fluid'])])]
    else:
        # fluid and wall at random; the WCSPH Group's pairs: no wall <- wall
        wall = rs.uniform(size=n) < 0.35
        arr = [('fluid', X[~wall], H[~wall]), ('wall', X[wall], H[wall])]
        mov = [moving[~wall], moving[wall]]
        groups = [(0, [('fluid', ['fluid', 'wall']), ('wall', ['fluid'])])]
        order = np.concatenate([np.flatnonzero(~wall), np.flatnonzero(wall)])
        states = [(dX[order], dH) for dX, dH in states]
    L = Lists(monkeypatch, dim, arr, groups, zorder=zorder, records=records, moving=mov,
              extra_states=states)
    where = np.argsort(order)                   # original index -> index in L.X
    _assert_crossings(L, where[len(lat)::2], where[len(lat) + 1::2])
    L.check()
    return L, [s[0] for s in states]


# ---- 1. the skin shell ------------------------------------------------------------------------
def check_skin_shell(monkeypatch, dim, zorder):
    """pairs at k h + f S, f in F_SHELL, across faces, edges and corners of the cell grid; each
    member moves towards its partner by 0.25 S, then by 0.235 S more (drift 0.97 S): both
    reuse the build, every pair with 2 x (its approach) > f S is now in the support"""
    L, states = _shell_case(monkeypatch, dim, zorder)
    S = L.S
    prev = np.zeros_like(L.X)
    for dX, a in zip(states, (0.25, 0.485)):
        L.move(dX - prev, path='reuse', need=2 * a * S)
        prev = dX
    return L


# ---- 2. growing and unequal h -----------------------------------------------------------------
def check_growing_h(monkeypatch, dim, zorder, seed=5):
    """(a) destinations whose h grows by dh while they and their partners approach by d:
    2 d + k dh = 0.97 S (deferred check: confirm() is False); the partner has a smaller h, so
    only the destination's half of the accept test takes the pair.  (b) pairs h_i = 0.8 h_j at
    k h_j + f S (f < 0 too): only the r^2 < (k h_j)^2 half accepts them, in the build (the small
    particle's list) and in the consumer.  Then h grows on until 2 d + k dh = 1.02 S: a
    rebuild."""
    rs = np.random.RandomState(seed)
    kr = 2.0
    h0 = HDX * DX
    lat = _lattice(dim, NSIDE[dim], rs)
    Hl = h0 * rs.uniform(0.85, 1.0, len(lat))
    Hl[0] = h0                                 # hmax, whatever grows below
    S = SKIN * kr * h0
    d = 0.25 * S
    dh = (0.97 * S - 2 * d) / kr
    lo, hi = lat.min(axis=0), lat.max(axis=0)
    P, U, H, G = [], [], [], []
    dirs = _directions(dim)
    for kind, fs in (('grow', F_SHELL), ('small', (-0.5,) + F_SHELL)):
        for f in fs:
            for _ in range(3):
                e = dirs[rs.randint(len(dirs))]
                u = e / np.linalg.norm(e)
                mid = lo + (hi - lo) * rs.uniform(0.2, 0.8, 3)
                mid[dim:] = 0.0
                if kind == 'grow':
                    hi_, hj_ = 0.95 * h0 - dh, 0.85 * h0
                    r = kr * hi_ + f * S
                else:
                    hi_, hj_ = 0.8 * h0, h0
                    r = kr * hj_ + f * S
                P += [mid - 0.5 * r * u, mid + 0.5 * r * u]
                U.append(u)
                H += [hi_, hj_]
                G += [kind == 'grow', False]
    P, U, H, G = np.array(P), np.array(U), np.array(H), np.array(G)
    n = len(lat) + len(P)
    X = np.concatenate([lat, P])
    Hall = np.concatenate([Hl, H])
    moving = np.zeros(n, dtype=bool)
    moving[len(lat):] = True
    dX = np.zeros((n, 3))
    dX[len(lat):] = _toward(U, d)
    dH = np.zeros(n)
    dH[len(lat):][G] = dh
    dh2 = 0.05 * S / kr
    dH2 = np.where(dH > 0, dh2, 0.0)
    L = Lists(monkeypatch, dim, [('fluid', X, Hall)], [(0, [('fluid', ['fluid'])])],
              zorder=zorder, moving=[moving], extra_states=[(dX, dH), (dX, dH + dH2)])
    L.check()
    L.move(dX, dH, path='reuse', need=0.97 * S, deferred=True)
    L.move(0.0, dH2, path='rebuild', need=1.02 * S)
    return L


# ---- 3. past the limit ------------------------------------------------------------------------
def check_past_the_limit(monkeypatch, dim, zorder):
    """a drift of 0.99 S: a full build, exact after it; the same again from the new build
    through update(deferred=True), an evaluation and confirm()"""
    L, states = _shell_case(monkeypatch, dim, zorder, moves=(0.495, 0.99))
    S = L.S
    L.move(states[0], path='rebuild', need=0.99 * S)
    L.move(states[1] - states[0], path='rebuild', need=0.99 * S, deferred=True)
    return L


# ---- 4. periodic ------------------------------------------------------------------------------
def _patterns(dim):
    return [p + (0,) * (3 - dim) for p in itertools.product((0, 1), repeat=dim) if any(p)]


def check_periodic(monkeypatch, dim, pattern, ncase, zorder):
    """a box periodic along `pattern`, with 1, 2 or 3 internal cells along a periodic axis (axis
    a gets 1 + (ncase + a) % 3), a jittered lattice filling it and pairs in the skin shell
    across the periodic boundary, moved towards each other until the drift is 0.97 S"""
    rs = np.random.RandomState(17 + ncase)
    kr, h = 2.0, HDX * DX
    S = SKIN * kr * h
    cell = kr * h + S
    lo, hi = np.zeros(3), np.zeros(3)
    for a in range(dim):
        if pattern[a]:
            nc = 1 + (ncase + a) % 3
            hi[a] = (nc + 0.5) * cell
        else:
            hi[a] = 8 * DX
    m = np.maximum(np.round((hi - lo) / DX).astype(int), 1)
    axes = [(np.arange(m[a]) + 0.5) * (hi[a] - lo[a]) / m[a] if a < dim else np.zeros(1)
            for a in range(3)]
    lat = np.stack(np.meshgrid(*axes, indexing='ij'), axis=-1).reshape(-1, 3)
    lat[:, :dim] += 0.2 * DX * rs.uniform(-1, 1, (len(lat), dim))
    for a in range(dim):
        if pattern[a]:
            lat[:, a] = np.mod(lat[:, a] - lo[a], hi[a] - lo[a]) + lo[a]
        else:
            lat[:, a] = np.clip(lat[:, a], lo[a], hi[a])
    # pairs across the boundary: midpoint on lo of the periodic axes the direction crosses
    P, U = [], []
    for e in _directions(dim):
        if not any(e[a] and pattern[a] for a in range(3)):
            continue
        u = e / np.linalg.norm(e)
        for f in (0.3, 0.95):
            mid = lo + (hi - lo) * rs.uniform(0.3, 0.7, 3)
            for a in range(dim):
                if e[a] and pattern[a]:
                    mid[a] = lo[a]
            mid[dim:] = 0.0
            r = kr * h + f * S
            p = np.array([mid - 0.5 * r * u, mid + 0.5 * r * u])
            for a in range(dim):
                if pattern[a]:
                    p[:, a] = np.mod(p[:, a] - lo[a], hi[a] - lo[a]) + lo[a]
            P += list(p)
            U.append(u)
    P, U = np.array(P), np.array(U)
    X = np.concatenate([lat, P])
    n = len(X)
    moving = np.zeros(n, dtype=bool)
    moving[len(lat):] = True
    dX = np.zeros((n, 3))
    dX[len(lat):] = _toward(U, 0.485 * S)
    # the moved members stay inside the box (the library wraps positions only at a build)
    Y = X + dX
    for a in range(dim):
        if pattern[a]:
            assert np.all((Y[:, a] > lo[a]) & (Y[:, a] < hi[a]))
    L = Lists(monkeypatch, dim, [('fluid', X, np.full(n, h))], [(0, [('fluid', ['fluid'])])],
              box=(lo, hi, pattern), zorder=zorder, moving=[moving], extra_states=[(dX, 0.0)])
    assert L.S == pytest.approx(S, rel=1e-12)
    L.check()
    L.move(dX, path='reuse', need=0.97 * S)
    return L


# ---- 5. warps, tiles and capacity -------------------------------------------------------------
def check_crowds(monkeypatch, dim, zorder, seed=23):
    """one case with: a dense cluster (more than LB_TILE = 128 candidates in one row segment, so
    the tile loop of k_list_build runs several times), a sparse block (rows of fewer than 32
    particles: one warp serves several rows), an isolated particle and two coincident ones; the
    approach pairs of the skin shell move to a drift of 0.97 S."""
    rs = np.random.RandomState(seed)
    kr, h = 2.0, HDX * DX
    S = SKIN * kr * h
    cell = kr * h + S
    lat = _lattice(dim, {1: 24, 2: 14, 3: 12}[dim], rs)
    ext = lat.max(axis=0)
    # a sparse block beyond +y (+x in 1-D), spacing 2 dx: the rows through it are short
    ax = 1 if dim > 1 else 0
    sp = _lattice(dim, {1: 6, 2: 5, 3: 4}[dim], rs, dx=2 * DX, jitter=0.1)
    sp[:, ax] += ext[ax] + 3 * DX
    # a dense cluster: 140 particles in a cube of edge 0.6 cell inside the lattice
    cl = np.zeros((140, 3))
    cl[:, :dim] = 0.5 * ext[:dim] + 0.6 * cell * rs.uniform(-0.5, 0.5, (140, dim))
    # isolated: beyond the reach of all; coincident: two at one point
    iso = np.zeros((1, 3))
    iso[0, :dim] = -3 * cell
    co = np.zeros((2, 3))
    co[:, :dim] = 0.25 * ext[:dim] + 0.013
    X0 = np.concatenate([lat, sp, cl, iso, co])
    P, U = _approach_pairs(dim, X0, kr, h, rs, fs=(0.6, 0.95) if dim > 1 else F_SHELL,
                           within=(lat.min(axis=0), lat.max(axis=0)))
    X = np.concatenate([X0, P])
    n = len(X)
    moving = np.zeros(n, dtype=bool)
    moving[len(X0):] = True
    i_iso = len(lat) + len(sp) + len(cl)
    keep = np.zeros(n, dtype=bool)
    keep[[i_iso + 1, i_iso + 2]] = True          # the coincident pair is never nudged apart
    dX = np.zeros((n, 3))
    dX[len(X0):] = _toward(U, 0.485 * S)
    L = Lists(monkeypatch, dim, [('fluid', X, np.full(n, h))], [(0, [('fluid', ['fluid'])])],
              zorder=zorder, moving=[moving], keep=[keep], extra_states=[(dX, 0.0)])
    assert np.array_equal(L.X[i_iso + 1], L.X[i_iso + 2])
    _assert_crossings(L, np.arange(len(X0), n, 2), np.arange(len(X0) + 1, n, 2))
    sig = L.signature()[0]
    assert sig[0][i_iso] == 1 and sig[1][i_iso] == L.key[i_iso]       # itself only
    assert sig[0][i_iso + 1] == sig[0][i_iso + 2] >= 2
    assert L.check()[0] > 0
    L.move(dX, path='reuse', need=0.97 * S)
    return L


def check_capacity(monkeypatch, dim, zorder, seed=37):
    """a block of the lattice compressed to `factor` times its density (3; 8 in 1-D, where
    three times the few neighbours still fits the head-room of the list length): the rebuild
    outgrows the entries reserved per destination and regrows them"""
    rs = np.random.RandomState(seed)
    kr, h = 2.0, HDX * DX
    cell = kr * h * (1 + SKIN)
    lat = _lattice(dim, {1: 40, 2: 16, 3: 11}[dim], rs)
    ext = lat.max(axis=0)
    n = len(lat)
    c = 0.4 * ext
    blk = np.all(np.abs(lat[:, :dim] - c[:dim]) < (4.0 if dim == 1 else 2.0) * cell, axis=1)
    factor = 8.0 if dim == 1 else 3.0
    comp = np.zeros((n, 3))
    comp[blk] = (c - lat[blk]) * (1.0 - factor ** (-1.0 / dim))
    comp[:, dim:] = 0.0
    L = Lists(monkeypatch, dim, [('fluid', lat, np.full(n, h))], [(0, [('fluid', ['fluid'])])],
              zorder=zorder, moving=[blk], extra_states=[(comp, 0.0)])
    L.check()
    cap0 = L.stats()['list_entries_per_particle']
    assert L.reference()[0].sum(axis=1).max() <= cap0
    L.move(comp, path='rebuild')
    cap1 = L.stats()['list_entries_per_particle']
    assert cap1 > cap0, (cap0, cap1)
    # the exact test alone already needs more than the old length
    assert L.reference()[0].sum(axis=1).max() > cap0
    return L


def check_one_cell(monkeypatch, dim, zorder, seed=29):
    """every particle in one cell: every pair is accepted; a move within the skin reuses"""
    rs = np.random.RandomState(seed)
    kr, h = 2.0, HDX * DX
    S = SKIN * kr * h
    n = 60
    X = np.zeros((n, 3))
    X[:, :dim] = 0.45 * kr * h * rs.uniform(0, 1, (n, dim))
    dX = np.zeros((n, 3))
    dX[:, :dim] = 0.3 * S * rs.uniform(-1, 1, (n, dim)) / np.sqrt(dim)
    L = Lists(monkeypatch, dim, [('fluid', X, np.full(n, h))], [(0, [('fluid', ['fluid'])])],
              zorder=zorder, extra_states=[(dX, 0.0)])
    pairs = L.check()
    assert pairs == [n * n]
    L.move(dX, path='reuse')
    return L


# ---- 6. what the lists are filtered for --------------------------------------------------------
def check_two_groups(monkeypatch, dim, zorder, seed=31):
    """two generic Groups on different (destination, source) sets, one after the other: the
    second is not covered by the lists the first built and forces a rebuild with the union (at
    least one: how many depends on how the Group's destinations are launched); both stay exact
    through a move that reuses the build, which rebuilds nothing"""
    rs = np.random.RandomState(seed)
    kr, h = 2.0, HDX * DX
    S = SKIN * kr * h
    lat = _lattice(dim, {1: 30, 2: 16, 3: 11}[dim], rs)
    lab = rs.randint(0, 3, len(lat))
    n = len(lat)
    dX = np.zeros((n, 3))
    dX[:, :dim] = 0.4 * S * rs.uniform(-1, 1, (n, dim)) / np.sqrt(dim)
    arrays = [(nm, lat[lab == k], np.full(int((lab == k).sum()), h))
              for k, nm in enumerate(('a', 'b', 'c'))]
    order = np.concatenate([np.flatnonzero(lab == k) for k in range(3)])
    groups = [(0, [('a', ['a', 'b'])]), (1, [('b', ['a', 'c']), ('c', ['c'])])]
    L = Lists(monkeypatch, dim, arrays, groups, zorder=zorder,
              extra_states=[(dX[order], 0.0)])
    st0 = L.stats()
    L.check()
    st1 = L.stats()
    # the positions did not change: one build serves the first Group, every further one was
    # forced by the second
    assert st1['list_builds'] - st0['list_builds'] >= 2, (st0['list_builds'], st1['list_builds'])
    L.move(dX[order], path='reuse')
    st2 = L.stats()
    assert st2['list_builds'] == st1['list_builds']
    return L


# ---- 7. the hand-written consumers on the moved state -------------------------------------------
def _pair_pass_count(L, dim):
    """b200sph_pair_pass with the WCSPH Group's equations (continuity, momentum and XSPH for
    fluid <- fluid, continuity and momentum for fluid <- wall, continuity for wall <- fluid):
    returns (pairs, launches on the 32-byte records)"""
    from pysph_b200 import _lib
    be = L.be
    n0 = be.stats()['pair_launches_r32']
    prog = _lib.PairProgram()
    CONT, MOM, XSPH = _lib.EQ_CONTINUITY, _lib.EQ_MOMENTUM, _lib.EQ_XSPH
    for (d, s), bits in {(0, 0): CONT | MOM | XSPH, (0, 1): CONT | MOM, (1, 0): CONT}.items():
        prog.eqmask[d][s] = bits
    prog.c0, prog.alpha, prog.beta, prog.eps_xsph = C0, 0.25, 0.0, 0.5
    for a in range(len(L.pas)):
        be.ctx.call('b200sph_eos', a, 0, RHO0, C0, 7.0, 0.0, 0)
    pairs = C.c_int64()
    be.ctx.call('b200sph_pair_pass', C.byref(prog), C.byref(pairs))
    return pairs.value, be.stats()['pair_launches_r32'] - n0


def check_pair_pass(monkeypatch, dim, records, zorder=0):
    """fluid and wall particles of the skin-shell case: the pair count of the pair pass (32- or
    48-byte records) equals the brute force's over the WCSPH Group's pairs, after the build and
    after each move in the skin; the generic signature on the same lists stays exact"""
    L, states = _shell_case(monkeypatch, dim, zorder, records=records, arrays=2)
    prev = np.zeros_like(L.X)
    want = L.check()
    for k, dX in enumerate([None] + states):
        if dX is not None:
            want = L.move(dX - prev, path='reuse')
            prev = dX
        pairs, r32 = _pair_pass_count(L, dim)
        assert r32 == (1 if records == '32' else 0)
        assert pairs == want[0], (k, pairs, want[0])
    return L


class Consumer(object):
    """The particles of L, in the same arrays, in a context of their own (the same fixed skin)
    whose Groups -- a scheme's -- run on a hand-written list consumer; `make(name, sl)` makes
    the particle array of L's array `name` from L's particles `sl`.  pairs() pushes L's current
    positions, updates (the path must be L's) and returns the evaluation's pair count."""

    def __init__(self, L, make, equations, kind):
        import pysph_b200 as pb
        self.L = L
        self.pas = [make(name, slice(L.start[k], L.start[k + 1]))
                    for k, name in enumerate(L.names)]
        self.ae = pb.B200AccelerationEval(self.pas, equations, L.kernel)
        assert [o[0] for o in self.ae.ops] == [kind], self.ae.ops
        self.prog = self.ae.ops[0][1]
        self.nn = pb.B200NNPS(L.dim, self.pas, backend=self.ae.backend, kernel=L.kernel)
        self.ae.set_nnps(self.nn)
        self.ae.count_pairs = True

    def pairs(self, path=None):
        be = self.ae.backend
        if path is not None:
            for k, pa in enumerate(self.pas):
                sl = slice(self.L.start[k], self.L.start[k + 1])
                pa.x[:], pa.y[:], pa.z[:] = self.L.X[sl, 0], self.L.X[sl, 1], self.L.X[sl, 2]
                be.push(k, ['x', 'y', 'z'])
            st0 = be.stats()
            self.nn.update()
            st1 = be.stats()
            assert (st1['light_updates'] - st0['light_updates'],
                    st1['full_builds'] - st0['full_builds']) == ((1, 0) if path == 'reuse' else (0, 1))
        self.ae.compute(0.0, 1e-5)
        return self.ae.last_pairs


def _accepted(L, dests, sources):
    """the brute force's pairs (destination of an array in `dests`, source of one in `sources`)"""
    cnt = L.reference()[0]
    rows = np.isin(L.owner, [L.names.index(d) for d in dests])
    return int(cnt[rows][:, [L.names.index(s) for s in sources]].sum())


def _consumer_moves(L, states, con, want):
    """the pair count of `con` after the build and after each reuse move of the skin shell;
    want(L) -> the count the brute force gives for the current positions"""
    assert con.pairs() == want(L) > 0
    prev = np.zeros_like(L.X)
    for k, dX in enumerate(states):
        L.move(dX - prev, path='reuse')
        prev = dX
        got = con.pairs(path='reuse')
        assert got == want(L), (k, got, want(L))


def check_tvf_pass(monkeypatch, dim):
    """EDACScheme(['fluid'], ['wall']) (transport velocity, solid walls) on the fluid and wall
    particles of the skin-shell case: the pair count of b200sph_tvf_pass equals the brute
    force's over the pairs its stages walk -- group 1 on the fluid and on the walls, the average
    pressure on the fluid, group 2 on the fluid, every one with fluid and walls as sources --
    after the build and after each move in the skin"""
    import pysph_b200 as pb
    L, states = _shell_case(monkeypatch, dim, 0, arrays=2)
    h, m, rho0 = HDX * DX, DX ** dim, 1.0

    def make(name, sl):
        f = pb.get_particle_array_edac if name == 'fluid' else pb.get_particle_array_edac_wall
        n = sl.stop - sl.start
        return f(name=name, x=L.X[sl, 0].copy(), y=L.X[sl, 1].copy(), z=L.X[sl, 2].copy(),
                 h=np.full(n, h), m=np.full(n, m * rho0), rho=np.full(n, rho0))
    sch = pb.EDACScheme(['fluid'], ['wall'], dim=dim, c0=10.0, nu=0.01, rho0=rho0,
                        pb=100.0, h=h, alpha=0.1, bql=True)
    con = Consumer(L, make, sch.get_equations(), 'tvf')
    passes = con.prog.passes
    assert passes == 7, passes

    def want(L):
        fl, wl = _accepted(L, ['fluid'], L.names), _accepted(L, ['wall'], L.names)
        return (fl + wl) * bool(passes & 1) + fl * bool(passes & 4) + fl * bool(passes & 2)
    _consumer_moves(L, states, con, want)
    return L


def check_solid_pass(monkeypatch, dim):
    """ElasticSolidsScheme on the particles of the skin-shell case as one elastic body: the pair
    count of b200sph_solid_pass equals the brute force's over both of its groups (every
    elastic particle a destination and a source), after the build and after each move"""
    import pysph_b200 as pb
    L, states = _shell_case(monkeypatch, dim, 0)
    h, rho0 = HDX * DX, 1.0

    def make(name, sl):
        n = sl.stop - sl.start
        return pb.get_particle_array_elastic_dynamics(
            name=name, x=L.X[sl, 0].copy(), y=L.X[sl, 1].copy(), z=L.X[sl, 2].copy(),
            h=np.full(n, h), m=np.full(n, rho0 * DX ** dim), rho=np.full(n, rho0),
            constants=dict(wdeltap=1.0, n=4, rho_ref=rho0, E=1e7, nu=0.3975))
    sch = pb.ElasticSolidsScheme(L.names, [], dim=dim)
    con = Consumer(L, make, sch.get_equations(), 'solid')
    passes = con.prog.passes
    assert passes == 3, passes

    def want(L):
        return _accepted(L, L.names, L.names) * (bool(passes & 1) + bool(passes & 2))
    _consumer_moves(L, states, con, want)
    return L


# ---- the tests --------------------------------------------------------------------------------
DIMS = [1, 2, 3]
ZORDER = [(1, 0), (2, 0), (2, 1), (3, 0), (3, 1)]       # (dim, zorder): rows exist in 2-D / 3-D
PERIODIC = [(dim, p, nc, z) for dim in DIMS for p in _patterns(dim) for nc in (0, 1, 2)
            for z in ((0,) if dim == 1 else (nc % 2,))]


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_skin_shell(monkeypatch, dim, zorder):
    check_skin_shell(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_growing_and_unequal_h(monkeypatch, dim, zorder):
    check_growing_h(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_past_the_limit(monkeypatch, dim, zorder):
    check_past_the_limit(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,pattern,ncase,zorder', PERIODIC)
def test_periodic(monkeypatch, dim, pattern, ncase, zorder):
    check_periodic(monkeypatch, dim, pattern, ncase, zorder)


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_crowds_tiles_and_capacity(monkeypatch, dim, zorder):
    check_crowds(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_capacity_regrows(monkeypatch, dim, zorder):
    check_capacity(monkeypatch, dim, zorder)


@pytest.mark.parametrize('dim', DIMS)
def test_all_in_one_cell(monkeypatch, dim):
    check_one_cell(monkeypatch, dim, 0)


@pytest.mark.parametrize('dim,zorder', ZORDER)
def test_two_groups_force_the_union(monkeypatch, dim, zorder):
    check_two_groups(monkeypatch, dim, zorder)


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('dim', [2, 3])
def test_pair_pass_counts(monkeypatch, dim, records):
    check_pair_pass(monkeypatch, dim, records)


@pytest.mark.parametrize('dim', [2, 3])
def test_tvf_pass_counts(monkeypatch, dim):
    check_tvf_pass(monkeypatch, dim)


@pytest.mark.parametrize('dim', [2, 3])
def test_solid_pass_counts(monkeypatch, dim):
    check_solid_pass(monkeypatch, dim)
