"""ctypes wrapper + WCSPH driver for the fp64 CPU oracle (liboracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  Nothing in pysph_b200/ may
import this module.

The driver below restates, independently of pysph_b200.program, which loops the
reference runs for a WCSPHScheme (pysph/sph/scheme.py:388-506), in which order
(pysph/sph/integrator.py:344-361 PEC, :401-420 EPEC) and how the solver picks
the time step (pysph/solver/solver.py:454-507, :647-688;
pysph/sph/integrator.py:161-200).

Pinned to the reference: see oracle/README.md and DESIGN.md section 5.  One function is
NOT: ``mirror_ghosts`` (a restatement of nnps_base.pyx:506-689; parity unpinned -- the
reference holds no mirror fixture and its DomainManager cannot be executed here).
"""
import ctypes as C
import os
import subprocess
from math import sqrt

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, 'liboracle.so')

MAX_ARRAYS = 8
K_IDS = {'CubicSpline': 0, 'WendlandQuintic': 1, 'QuinticSpline': 2,
         'Gaussian': 3}
EQ_SUMDENS, EQ_CONT, EQ_MOM, EQ_XSPH, EQ_AV, EQ_LAMINAR = 1, 2, 4, 8, 16, 32

_PTR_FIELDS = ['x', 'y', 'z', 'h', 'm', 'rho', 'u', 'v', 'w', 'p', 'cs',
               'arho', 'au', 'av', 'aw', 'ax', 'ay', 'az', 'dt_cfl',
               'dt_force', 'x0', 'y0', 'z0', 'u0', 'v0', 'w0', 'rho0',
               'uhat', 'vhat', 'what', 'V', 'pavg', 'nnbr', 'auhat', 'avhat',
               'awhat', 'ap', 'p0']
TVF_PGRAD, TVF_AV, TVF_VISC, TVF_ASTRESS, TVF_EDAC, TVF_NOSLIP = 1, 2, 4, 8, 16, 32
TVF_MOM, TVF_XSPH = 64, 128
# elastic dynamics (solid_mech/basic.py:52-59), in the order of orc_array
_SYM = ['00', '01', '02', '11', '12', '22']
_PTR_FIELDS += ['v%d%d' % (i, j) for i in range(3) for j in range(3)] + \
    ['s' + k for k in _SYM] + ['as' + k for k in _SYM] + ['r' + k for k in _SYM] + \
    ['s' + k + '0' for k in _SYM] + ['e', 'e0', 'ae']
# wall arrays of the EDAC scheme (wc/edac.py:752-753); the C field of 'vg' is 'vgw'
_PTR_FIELDS += ['wij', 'uf', 'vf', 'wf', 'ug', 'vgw', 'wg']


class OrcArray(C.Structure):
    _fields_ = [('n', C.c_int64), ('n_real', C.c_int64)] + \
        [(f, C.POINTER(C.c_double)) for f in _PTR_FIELDS]


class OrcPairProgram(C.Structure):
    _fields_ = [('kernel', C.c_int), ('dim', C.c_int),
                ('c0', C.c_double), ('alpha', C.c_double), ('beta', C.c_double),
                ('gx', C.c_double), ('gy', C.c_double), ('gz', C.c_double),
                ('tensile_correction', C.c_int),
                ('eps_xsph', C.c_double),
                ('real_only', C.c_int),
                ('eqmask', (C.c_uint32 * MAX_ARRAYS) * MAX_ARRAYS),
                ('src_order', (C.c_int * MAX_ARRAYS) * MAX_ARRAYS),
                ('dest_order', C.c_int * MAX_ARRAYS),
                ('nu', C.c_double), ('eta', C.c_double)]


class OrcTvfProgram(C.Structure):
    _fields_ = [('kernel', C.c_int), ('dim', C.c_int),
                ('fluid_mask', C.c_uint32), ('bql', C.c_int),
                ('eqbits', C.c_uint32),
                ('pb', C.c_double), ('nu', C.c_double), ('edac_nu', C.c_double),
                ('c0', C.c_double), ('rho0', C.c_double), ('alpha', C.c_double),
                ('gx', C.c_double), ('gy', C.c_double), ('gz', C.c_double),
                ('tdamp', C.c_double), ('t', C.c_double), ('solid_mask', C.c_uint32),
                ('eps_xsph', C.c_double), ('clamp_p', C.c_int)]


class OrcSolidProgram(C.Structure):
    _fields_ = [('kernel', C.c_int), ('dim', C.c_int),
                ('elastic_mask', C.c_uint32), ('source_mask', C.c_uint32),
                ('grad3d', C.c_int), ('eps', C.c_double),
                ('alpha', C.c_double), ('beta', C.c_double), ('eps_xsph', C.c_double),
                ('c0_ref', C.c_double * MAX_ARRAYS), ('rho_ref', C.c_double * MAX_ARRAYS),
                ('wdeltap', C.c_double * MAX_ARRAYS), ('n', C.c_double * MAX_ARRAYS),
                ('G', C.c_double * MAX_ARRAYS)]


def build(force=False):
    src = os.path.join(HERE, 'sph_oracle.c')
    if force or not os.path.exists(LIB) or \
            os.path.getmtime(LIB) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', HERE, 'liboracle.so'],
                              stdout=subprocess.DEVNULL)
    return LIB


_lib = None


def load():
    global _lib
    if _lib is None:
        build()
        lib = C.CDLL(LIB)
        lib.orc_create.restype = C.c_void_p
        lib.orc_create.argtypes = [C.c_int, C.c_int, C.c_double]
        lib.orc_destroy.argtypes = [C.c_void_p]
        lib.orc_set_array.argtypes = [C.c_void_p, C.c_int, C.POINTER(OrcArray)]
        lib.orc_set_num_threads.argtypes = [C.c_int]
        lib.orc_get_max_threads.restype = C.c_int
        lib.orc_update_domain.argtypes = [C.c_void_p]
        lib.orc_nnps_update.argtypes = [C.c_void_p]
        lib.orc_nnps_update.restype = C.c_int
        lib.orc_get_grid.argtypes = [C.c_void_p] + [C.c_void_p] * 6
        for f in ('orc_find_neighbors', 'orc_brute_neighbors'):
            getattr(lib, f).restype = C.c_int64
            getattr(lib, f).argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64,
                                        C.c_void_p, C.c_int64]
        lib.orc_eos.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double,
                                C.c_double, C.c_double, C.c_double, C.c_int]
        lib.orc_ferrari_h.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_int,
                                      C.c_int]
        lib.orc_pair_pass.restype = C.c_int64
        lib.orc_pair_pass.argtypes = [C.c_void_p, C.POINTER(OrcPairProgram)]
        lib.orc_stage.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
        lib.orc_dt_factors.argtypes = [C.c_void_p, C.c_void_p]
        for f in ('orc_tvf_pass1', 'orc_tvf_pass2', 'orc_tvf_wall', 'orc_tvf_avgp'):
            getattr(lib, f).restype = C.c_int64
            getattr(lib, f).argtypes = [C.c_void_p, C.POINTER(OrcTvfProgram)]
        lib.orc_stage_tvf.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
        lib.orc_stage_edac.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
        for f in ('orc_solid_group1', 'orc_solid_group2'):
            getattr(lib, f).restype = C.c_int64
            getattr(lib, f).argtypes = [C.c_void_p, C.POINTER(OrcSolidProgram)]
        lib.orc_stage_solid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
        lib.orc_eigen_sym3.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.orc_kernel_w.restype = C.c_double
        lib.orc_kernel_w.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double]
        lib.orc_kernel_grad.argtypes = [C.c_int, C.c_int, C.c_void_p,
                                        C.c_double, C.c_double, C.c_void_p]
        lib.orc_kernel_deltap.restype = C.c_double
        lib.orc_kernel_deltap.argtypes = [C.c_int]
        lib.orc_kernel_radius_scale.restype = C.c_double
        lib.orc_kernel_radius_scale.argtypes = [C.c_int]
        _lib = lib
    return _lib


def eigen_sym3(a):
    """(eigenvalues[3], eigenvectors as columns [3,3]) of a symmetric 3x3 matrix."""
    a = np.ascontiguousarray(a, dtype=np.float64).reshape(9)
    v = np.zeros(9)
    d = np.zeros(3)
    load().orc_eigen_sym3(a.ctypes.data, v.ctypes.data, d.ctypes.data)
    return d, v.reshape(3, 3)


def kernel_w(kernel, dim, rij, h):
    return load().orc_kernel_w(K_IDS[kernel], dim, rij, h)


def kernel_grad(kernel, dim, xij, rij, h):
    x = (C.c_double * 3)(*xij)
    g = (C.c_double * 3)()
    load().orc_kernel_grad(K_IDS[kernel], dim, x, rij, h, g)
    return np.array(g[:])


class Oracle(object):
    """fp64 evaluator over a list of host particle arrays (any object with
    ``properties`` dict of float64 numpy arrays, ``get_number_of_particles``
    and ``num_real_particles``).  Operates IN PLACE on those arrays."""

    def __init__(self, particle_arrays, dim, kernel='CubicSpline',
                 radius_scale=None, threads=1):
        self.lib = load()
        self.pas = list(particle_arrays)
        self.names = [pa.name for pa in self.pas]
        self.index = dict((n, i) for i, n in enumerate(self.names))
        self.dim = dim
        self.kernel = kernel
        self.kid = K_IDS[kernel]
        if radius_scale is None:
            radius_scale = self.lib.orc_kernel_radius_scale(self.kid)
        self.radius_scale = radius_scale
        self.lib.orc_set_num_threads(int(threads))
        self.h = C.c_void_p(self.lib.orc_create(len(self.pas), dim,
                                                 radius_scale))
        self.bind()

    def bind(self):
        """(Re)bind host pointers -- call after any array was re-allocated."""
        self._keep = []
        for i, pa in enumerate(self.pas):
            oa = OrcArray()
            oa.n = pa.get_number_of_particles()
            oa.n_real = pa.get_number_of_particles(real=True)
            for f in _PTR_FIELDS:
                name = 'vg' if f == 'vgw' else f
                if name in pa.properties:
                    a = pa.properties[name]
                    assert a.dtype == np.float64 and a.flags.c_contiguous
                    setattr(oa, f, a.ctypes.data_as(C.POINTER(C.c_double)))
            self._keep.append(oa)
            self.lib.orc_set_array(self.h, i, C.byref(oa))

    def __del__(self):
        try:
            self.lib.orc_destroy(self.h)
        except Exception:
            pass

    # -- NNPS -----------------------------------------------------------------
    def update_domain(self):
        self.lib.orc_update_domain(self.h)

    def nnps_update(self):
        rc = self.lib.orc_nnps_update(self.h)
        if rc == -1:
            raise RuntimeError('ERROR: LinkedListNNPS requires too many cells')
        if rc == -3:
            raise FloatingPointError('oracle: non-finite particle positions (the run blew up)')
        if rc:
            raise RuntimeError('oracle nnps_update failed (%d)' % rc)

    def grid(self):
        cs, hm = C.c_double(), C.c_double()
        xmin, xmax = (C.c_double * 3)(), (C.c_double * 3)()
        nc, n = (C.c_int * 3)(), C.c_int64()
        self.lib.orc_get_grid(self.h, C.byref(cs), C.byref(hm), xmin, xmax, nc,
                              C.byref(n))
        return dict(cell_size=cs.value, hmin=hm.value, xmin=np.array(xmin[:]),
                    xmax=np.array(xmax[:]), ncells=np.array(nc[:]),
                    n_cells=n.value)

    def _nbrs(self, fn, dst, src, d_idx):
        cap = 4096
        while True:
            buf = np.empty(cap, dtype=np.uint32)
            n = fn(self.h, dst, src, int(d_idx), buf.ctypes.data, cap)
            if n <= cap:
                return buf[:n].copy()
            cap = int(n)

    def neighbors(self, dst, src, d_idx):
        return self._nbrs(self.lib.orc_find_neighbors, dst, src, d_idx)

    def brute_neighbors(self, dst, src, d_idx):
        return self._nbrs(self.lib.orc_brute_neighbors, dst, src, d_idx)

    # -- equations ------------------------------------------------------------
    def eos(self, arr, hg, rho0, c0, gamma, p0=0.0, real_only=False):
        self.lib.orc_eos(self.h, arr, int(hg), rho0, c0, gamma, p0,
                         int(real_only))

    def ferrari_h(self, arr, hdx, dim, real_only=False):
        self.lib.orc_ferrari_h(self.h, arr, hdx, dim, int(real_only))

    def pair_pass(self, eqs, real_only=True, c0=0.0, alpha=0.0, beta=0.0,
                  gx=0.0, gy=0.0, gz=0.0, tensile_correction=False,
                  eps_xsph=0.5, nu=0.0, eta=0.01):
        """eqs: list of (bit, dest_index, [source indices]) in user order."""
        P = OrcPairProgram()
        P.nu, P.eta = nu, eta
        P.kernel, P.dim = self.kid, self.dim
        P.c0, P.alpha, P.beta = c0, alpha, beta
        P.gx, P.gy, P.gz = gx, gy, gz
        P.tensile_correction = int(tensile_correction)
        P.eps_xsph = eps_xsph
        P.real_only = int(real_only)
        dests = []
        orders = {}
        for bit, d, srcs in eqs:
            if d not in dests:
                dests.append(d)
                orders[d] = []
            for s in srcs:
                P.eqmask[d][s] |= bit
                if s not in orders[d]:
                    orders[d].append(s)
        for d in range(MAX_ARRAYS):
            for k in range(MAX_ARRAYS):
                P.src_order[d][k] = -1
            P.dest_order[d] = -1
        for k, d in enumerate(dests):
            P.dest_order[k] = d
            for j, s in enumerate(orders[d]):
                P.src_order[d][j] = s
        return self.lib.orc_pair_pass(self.h, C.byref(P))

    def stage(self, arr, which, dt):
        self.lib.orc_stage(self.h, arr, which, dt)

    # -- EDAC, transport-velocity branch ---------------------------------------
    def tvf_program(self, fluids, eqbits, bql=True, pb=0.0, nu=0.0, edac_nu=0.0,
                    c0=0.0, rho0=0.0, alpha=0.0, gx=0.0, gy=0.0, gz=0.0,
                    tdamp=0.0, t=0.0, solids=(), eps_xsph=0.0, clamp_p=False):
        P = OrcTvfProgram()
        P.kernel, P.dim = self.kid, self.dim
        P.fluid_mask = sum(1 << f for f in fluids)
        P.solid_mask = sum(1 << f for f in solids)
        P.eps_xsph, P.clamp_p = eps_xsph, int(clamp_p)
        P.bql, P.eqbits = int(bql), eqbits
        P.pb, P.nu, P.edac_nu, P.c0, P.rho0, P.alpha = pb, nu, edac_nu, c0, rho0, alpha
        P.gx, P.gy, P.gz, P.tdamp, P.t = gx, gy, gz, tdamp, t
        return P

    def tvf_pass1(self, P):
        return self.lib.orc_tvf_pass1(self.h, C.byref(P))

    def tvf_pass2(self, P):
        return self.lib.orc_tvf_pass2(self.h, C.byref(P))

    def tvf_wall(self, P):
        return self.lib.orc_tvf_wall(self.h, C.byref(P))

    def tvf_avgp(self, P):
        return self.lib.orc_tvf_avgp(self.h, C.byref(P))

    def stage_tvf(self, arr, which, dt):
        self.lib.orc_stage_tvf(self.h, arr, which, dt)

    def stage_edac(self, arr, which, dt):
        self.lib.orc_stage_edac(self.h, arr, which, dt)

    # -- elastic dynamics -------------------------------------------------------
    def solid_program(self, elastic, sources, eps=0.3, alpha=1.0, beta=1.0,
                      eps_xsph=0.5, grad3d=False):
        P = OrcSolidProgram()
        P.kernel, P.dim = self.kid, self.dim
        P.elastic_mask = sum(1 << a for a in elastic)
        P.source_mask = sum(1 << a for a in sources)
        P.grad3d, P.eps = int(grad3d), eps
        P.alpha, P.beta, P.eps_xsph = alpha, beta, eps_xsph
        for a, pa in enumerate(self.pas):
            c = getattr(pa, 'constants', {})
            for k in ('c0_ref', 'rho_ref', 'wdeltap', 'n', 'G'):
                if k in c:
                    getattr(P, k)[a] = float(np.ravel(c[k])[0])
        return P

    def solid_group1(self, P):
        return self.lib.orc_solid_group1(self.h, C.byref(P))

    def solid_group2(self, P):
        return self.lib.orc_solid_group2(self.h, C.byref(P))

    def stage_solid(self, arr, which, dt):
        self.lib.orc_stage_solid(self.h, arr, which, dt)

    def dt_factors(self):
        out = (C.c_double * 3)()
        self.lib.orc_dt_factors(self.h, out)
        return out[0], out[1], out[2]


def periodic_box_wrap(pas, lo, hi, periodic):
    """_box_wrap_periodic, pysph/base/nnps_base.pyx:699-743 (in place)."""
    for pa in pas:
        for d, name in enumerate(('x', 'y', 'z')):
            if not periodic[d]:
                continue
            a = pa.properties[name]
            L = hi[d] - lo[d]
            a[a < lo[d]] += L
            a[a > hi[d]] -= L


def periodic_ghosts(pas, lo, hi, periodic, cell_size, n_layers=2.0, factory=None):
    """_create_ghosts_periodic, pysph/base/nnps_base.pyx:744-940: returns NEW
    arrays = real particles + their periodic images (tag Ghost = 2) appended,
    ``num_real_particles`` unchanged.  Images: x first; then y images of the
    real particles AND of the x images; then z images of everything so far."""
    from pysph_b200.particle_array import get_particle_array_wcsph
    width = n_layers * cell_size
    out = []
    for pa in pas:
        nr = pa.get_number_of_particles(real=True)
        props = dict((k, v[:nr].copy()) for k, v in pa.properties.items())
        ghosts = dict((k, v[:0].copy()) for k, v in props.items())

        def images(src, name, d):
            lo_sel = (src[name] - lo[d]) <= width
            hi_sel = (hi[d] - src[name]) <= width
            new = []
            for sel, shift in ((lo_sel, hi[d] - lo[d]), (hi_sel, -(hi[d] - lo[d]))):
                blk = dict((k, v[sel].copy()) for k, v in src.items())
                blk[name] = blk[name] + shift
                new.append(blk)
            return new

        def cat(parts):
            return dict((k, np.concatenate([p[k] for p in parts])) for k in props)

        for d, name in enumerate(('x', 'y', 'z')):
            if not periodic[d]:
                continue
            new = images(ghosts, name, d) + images(props, name, d)
            ghosts = cat([ghosts] + new)
        allp = cat([props, ghosts])
        fac = factory.get(pa.name) if isinstance(factory, dict) else factory   # per array, by name
        q = (fac or get_particle_array_wcsph)(name=pa.name, **allp)
        q.set_num_real_particles(nr)
        q.tag[nr:] = 2
        out.append(q)
    return out


def mirror_ghosts(pas, lo, hi, mirror, cell_size, n_layers=2.0, factory=None):
    """_create_ghosts_mirror, pysph/base/nnps_base.pyx:506-689: returns NEW arrays = real
    particles + their mirror images (tag Ghost = 2) appended.  Selection: (x - min) <=
    n_layers * cell_size / (max - x) <= n_layers * cell_size (:568-590); image position
    x + (-2 (x - min)) / x + 2 (max - x), normal velocity times -1 (:598-611); x images of
    the real particles first, then y images of the images so far (low, high) followed by
    the y images of the real particles (high, low) (:613-652), then z likewise (:654-689)."""
    from pysph_b200.particle_array import get_particle_array_wcsph
    width = n_layers * cell_size
    vel = ('u', 'v', 'w')
    out = []
    for pa in pas:
        nr = pa.get_number_of_particles(real=True)
        props = dict((k, v[:nr].copy()) for k, v in pa.properties.items())
        added = dict((k, v[:0].copy()) for k, v in props.items())

        def image(src, name, d, low):
            sel = ((src[name] - lo[d]) <= width) if low else ((hi[d] - src[name]) <= width)
            blk = dict((k, v[sel].copy()) for k, v in src.items())
            blk[name] = blk[name] + (-2.0 * (blk[name] - lo[d]) if low else 2.0 * (hi[d] - blk[name]))
            blk[vel[d]] = -1.0 * blk[vel[d]]
            return blk

        def cat(parts):
            return dict((k, np.concatenate([p[k] for p in parts])) for k in props)

        for d, name in enumerate(('x', 'y', 'z')):
            if not mirror[d]:
                continue
            if d == 0:
                new = [image(props, name, d, True), image(props, name, d, False)]
            else:
                # both corner blocks select from `added` as it was before this axis
                new = [image(added, name, d, True), image(added, name, d, False),
                       image(props, name, d, False), image(props, name, d, True)]
            added = cat([added] + new)
        allp = cat([props, added])
        q = (factory or get_particle_array_wcsph)(name=pa.name, **allp)
        q.set_num_real_particles(nr)
        q.tag[nr:] = 2
        out.append(q)
    return out


class WCSPHOracleSolver(object):
    """Runs a WCSPHScheme simulation with the oracle: scheme.py:388-506 for the
    loops, integrator.py:344-361/401-420 for the stage order, solver.py for the
    time step.  ``params`` as returned by pysph_b200.geometry.*_params."""

    def __init__(self, particles, params, kernel='CubicSpline', threads=1,
                 domain=None):
        """domain = (lo[3], hi[3], periodic[3][, mirror[3]]) or None.  With a periodic
        or mirror domain every ``update_domain`` re-creates the periodic ghost images
        (DomainManager.update, nnps_base.pyx:405-433), so ``self.pas`` (the
        arrays with ghosts) is replaced each time."""
        p = dict(params)
        self.p = p
        self.integrator = p.get('integrator', 'EPEC')
        self.dim = p['dim']
        self.domain = domain
        self.kernel = kernel
        self.threads = threads
        self.pas = list(particles)
        if domain is not None:
            self._reghost()
        else:
            self.o = Oracle(particles, self.dim, kernel, threads=threads)
        ix = self.o.index
        self.fluids = [ix[n] for n in p['fluids']]
        self.solids = [ix[n] for n in p['solids']]
        self.all = self.fluids + self.solids
        self.dt = p['dt0']
        self.cfl = p.get('cfl', 0.3)
        self.n_damp = p.get('n_damp', 0)
        self.adaptive = p.get('adaptive_timestep', True)
        self.t = 0.0
        self.count = 0
        self._damping_factor = 1.0
        self.pairs_last_eval = 0
        self.pairs_total = 0
        # NNPS constructor: domain.update(); update()  (linked_list_nnps.pyx:84-88)
        self.update_domain()
        self.o.nnps_update()
        self._initialised = False

    def _reghost(self):
        lo, hi, per = self.domain[:3]
        mir = self.domain[3] if len(self.domain) > 3 else (0, 0, 0)
        real = []
        from pysph_b200.particle_array import get_particle_array_wcsph
        for pa in self.pas:
            nr = pa.get_number_of_particles(real=True)
            q = get_particle_array_wcsph(name=pa.name, **dict(
                (k, v[:nr].copy()) for k, v in pa.properties.items()))
            q.set_num_real_particles(nr)
            real.append(q)
        k = load().orc_kernel_radius_scale(K_IDS[self.kernel])
        hmax = max(float(np.max(q.h)) for q in real if len(q.h))
        if any(per) and any(mir):
            raise NotImplementedError('oracle: mirror planes in a periodic domain')
        if any(per):
            periodic_box_wrap(real, lo, hi, per)
            real = periodic_ghosts(real, lo, hi, per, k * hmax)
        if any(mir):                       # DomainManager.update, nnps_base.pyx:471-480
            real = mirror_ghosts(real, lo, hi, mir, k * hmax)
        self.pas = real
        self.o = Oracle(self.pas, self.dim, self.kernel, threads=self.threads)

    def update_domain(self):
        if self.domain is not None:
            self._reghost()
        self.o.update_domain()

    # AccelerationEval.compute for the WCSPH groups
    def evaluate(self):
        p, o = self.p, self.o
        pairs = 0
        if p.get('summation_density', False):
            pairs += o.pair_pass([(EQ_SUMDENS, f, self.all) for f in self.fluids],
                                 real_only=False)
        for f in self.fluids:
            o.eos(f, 0, p['rho0'], p['c0'], p['gamma'], 0.0, real_only=False)
        for s in self.solids:
            o.eos(s, 1 if p.get('hg_correction', False) else 0, p['rho0'],
                  p['c0'], p['gamma'], 0.0, real_only=False)
        eqs = [(EQ_CONT, s, self.fluids) for s in self.solids]
        for f in self.fluids:
            if not p.get('summation_density', False):
                eqs.append((EQ_CONT, f, self.all))
            eqs.append((EQ_MOM, f, self.all))
            if abs(p.get('nu', 0.0)) > 1e-14:        # scheme.py:486-496: before XSPH
                eqs.append((EQ_LAMINAR, f, self.all))
            eqs.append((EQ_XSPH, f, [f]))
        pairs += o.pair_pass(
            eqs, real_only=True, c0=p['c0'], alpha=p.get('alpha', 0.1),
            beta=p.get('beta', 0.0), gx=p.get('gx', 0.0), gy=p.get('gy', 0.0),
            gz=p.get('gz', 0.0),
            tensile_correction=p.get('tensile_correction', False), eps_xsph=0.5,
            nu=p.get('nu', 0.0))
        if p.get('update_h', False):
            for f in self.fluids:
                o.ferrari_h(f, p['hdx'], self.dim, real_only=False)
        self.pairs_last_eval = pairs
        self.pairs_total += pairs
        return pairs

    def compute_accelerations(self):
        self.o.nnps_update()
        self.evaluate()

    def _stage(self, which, dt):
        for a in self.all:
            self.o.stage(a, which, dt)

    def one_timestep(self, dt):
        self._stage(0, 0.0)
        if self.integrator == 'EPEC':
            self.compute_accelerations()
        self._stage(1, dt)
        self.update_domain()
        self.compute_accelerations()
        self._stage(2, dt)
        self.update_domain()

    def _compute_timestep(self):
        undamped = self.dt / self._damping_factor
        if not self.adaptive:
            return undamped
        f_cfl, f_force, hmin = self.o.dt_factors()
        dt_cfl = dt_force = np.inf
        if f_cfl > 0:
            dt_cfl = hmin / f_cfl
        if f_force > 0:
            dt_force = sqrt(hmin / sqrt(f_force))
        dt_min = min(dt_cfl, dt_force)
        if dt_min <= 0.0 or np.isinf(dt_min):
            return undamped
        return self.cfl * dt_min

    def _get_timestep(self):
        # solver.py:756-776 (tf: the final time the last step lands on; eps :441, :488)
        tf = self.p.get('tf', np.inf)
        eps = np.finfo(float).eps * 2 * tf * max(self.count, 1) if np.isfinite(tf) else 0.0
        if abs(tf - self.t) < eps:
            return self.dt
        dt = self._compute_timestep()
        if self.count < self.n_damp and self.n_damp > 0:
            frac = (self.count + 1) / float(self.n_damp)
            self._damping_factor = 0.5 * (np.sin(np.pi * (-0.5 + frac)) + 1.0)
        else:
            self._damping_factor = 1.0
        dt = dt * self._damping_factor
        if (self.t + dt) > (tf - eps):
            dt = tf - self.t
        return dt

    def initialise(self):
        if not self._initialised:
            self.evaluate()                 # initial_acceleration, no NNPS update
            self.dt = self._get_timestep()
            self._initialised = True

    def step(self):
        self.initialise()
        self.one_timestep(self.dt)
        self.t += self.dt
        self.count += 1
        self.dt = self._get_timestep()

    def solve(self, max_steps):
        self.initialise()
        while self.count < max_steps:
            self.step()


def edac_eqbits(p):
    """Which equations EDACScheme._get_internal_flow_equations emits in its second group
    (wc/edac.py:842-878)."""
    if abs(p.get('pb', 0.0)) > 1e-14:       # use_tvf, wc/edac.py:651-655
        bits = TVF_PGRAD | TVF_ASTRESS | TVF_EDAC
    else:                                   # external flows, :882-971
        bits = TVF_MOM | TVF_EDAC | TVF_XSPH
    if p.get('alpha', 0.0) > 0.0:
        bits |= TVF_AV
    if p.get('nu', 0.0) > 0.0:
        bits |= TVF_VISC
        if p.get('solids'):
            bits |= TVF_NOSLIP
    return bits


def edac_nu(p):
    """EDACScheme._get_edac_nu / attributes_changed, wc/edac.py:651-655, :766-774."""
    art_nu = p.get('edac_alpha', 0.5) * p.get('h', 0.0) * p['c0'] / 8
    return art_nu if art_nu > 0 else p.get('nu', 0.0)


class EDACOracleSolver(object):
    """EDACScheme(fluids, solids=[], pb != 0) with PECIntegrator + EDACTVFStep and a
    fixed time step (the Taylor-Green set-up, pysph/examples/taylor_green.py:
    190-203): wc/edac.py:776-880 for the groups, integrator.py:344-361 for the
    stage order.  ``params``: dim, c0, rho0, nu, pb, h (for edac_alpha), alpha,
    edac_alpha, bql, gx.., tdamp, dt."""

    def __init__(self, particles, params, kernel='QuinticSpline', threads=1,
                 domain=None):
        self.p = dict(params)
        self.dim = self.p['dim']
        self.domain = domain
        self.kernel = kernel
        self.threads = threads
        self.pas = list(particles)
        self.dt = self.p['dt']
        self.t = 0.0
        self.count = 0
        self.pairs_last_eval = 0
        if domain is not None:
            self._reghost()
        else:
            self.o = Oracle(self.pas, self.dim, kernel, threads=threads)
        self.update_domain()
        self.o.nnps_update()
        self._initialised = False

    def _reghost(self):
        lo, hi, per = self.domain
        from pysph_b200.particle_array import get_particle_array_edac, get_particle_array_edac_wall
        walls = self.p.get('solids') or ()
        fac = dict((pa.name, get_particle_array_edac_wall if pa.name in walls
                    else get_particle_array_edac) for pa in self.pas)
        real = []
        for pa in self.pas:
            nr = pa.get_number_of_particles(real=True)
            real.append(fac[pa.name](name=pa.name, **dict(
                (k, v[:nr].copy()) for k, v in pa.properties.items())))
        periodic_box_wrap(real, lo, hi, per)
        k = load().orc_kernel_radius_scale(K_IDS[self.kernel])
        hmax = max(float(np.max(q.h)) for q in real if len(q.h))
        self.pas = periodic_ghosts(real, lo, hi, per, k * hmax, factory=fac)
        self.o = Oracle(self.pas, self.dim, self.kernel, threads=self.threads)

    def update_domain(self):
        if self.domain is not None:
            self._reghost()
        self.o.update_domain()

    def evaluate(self, t=None):
        p, o = self.p, self.o
        walls = [i for i, pa in enumerate(self.pas) if pa.name in (p.get('solids') or ())]
        fl = [i for i in range(len(self.pas)) if i not in walls]
        tvf = abs(p.get('pb', 0.0)) > 1e-14
        bql = p.get('bql', True) and tvf        # the external-flow branch has no average pressure
        P = o.tvf_program(fl, edac_eqbits(p), bql=bql and not walls, pb=p['pb'],
                          nu=p.get('nu', 0.0), edac_nu=edac_nu(p), c0=p['c0'],
                          rho0=p['rho0'], alpha=p.get('alpha', 0.0),
                          gx=p.get('gx', 0.0), gy=p.get('gy', 0.0), gz=p.get('gz', 0.0),
                          tdamp=p.get('tdamp', 0.0), t=self.t if t is None else t,
                          solids=walls, eps_xsph=p.get('eps', 0.0),
                          clamp_p=p.get('clamp_p', False) and not tvf)
        pairs = o.tvf_pass1(P)
        if walls:
            # group 1 continues with the wall arrays, then the average pressure has a
            # group of its own (wc/edac.py:815-842)
            pairs += o.tvf_wall(P)
            if bql:
                pairs += o.tvf_avgp(P)
        pairs += o.tvf_pass2(P)
        self.pairs_last_eval = pairs
        return pairs

    def initialise(self):
        if not self._initialised:
            self.evaluate()                 # Solver.solve -> initial_acceleration
            self._initialised = True

    def step(self):
        # PECIntegrator.one_timestep integrator.py:344-361
        self.initialise()
        # steppers exist for the fluids only (wc/edac.py:682-687): walls do not move
        fl = [i for i, pa in enumerate(self.pas) if pa.name not in (self.p.get('solids') or ())]
        # EDACTVFStep with the transport velocity, EDACStep without (wc/edac.py:682)
        # (self.o is replaced by update_domain() in a periodic domain: look the method up each time)
        name = 'stage_tvf' if abs(self.p.get('pb', 0.0)) > 1e-14 else 'stage_edac'
        for a in fl:
            getattr(self.o, name)(a, 0, 0.0)
        for a in fl:
            getattr(self.o, name)(a, 1, self.dt)
        self.update_domain()
        self.o.nnps_update()
        self.evaluate(self.t)               # a_eval.compute(c_integrator.t, ...) integrator.py:286
        for a in fl:
            getattr(self.o, name)(a, 2, self.dt)
        self.update_domain()
        self.t += self.dt
        self.count += 1


class ElasticOracleSolver(object):
    """ElasticSolidsScheme(elastic_solids, solids=[]) with SolidMechStep and a fixed
    time step (pysph/examples/solid_mech/rings.py:80-84: the scheme's default
    EPECIntegrator): solid_mech/basic.py:604-651 for the groups,
    integrator.py:401-420 for the stage order."""

    def __init__(self, particles, params, kernel='CubicSpline', threads=1):
        self.p = dict(params)
        self.pas = list(particles)
        self.o = Oracle(self.pas, self.p['dim'], kernel, threads=threads)
        self.dt = self.p['dt']
        self.t = 0.0
        self.count = 0
        self.integrator = self.p.get('integrator', 'EPEC')
        self.pairs_last_eval = 0
        self.o.update_domain()
        self.o.nnps_update()
        self._initialised = False

    def _elastic(self):
        """indices of the elastic arrays; params['solids'] names the rigid ones (sources of
        every pair equation, destinations of none, never stepped: solid_mech/basic.py:613,
        :653-684)"""
        rigid = set(self.p.get('solids', ()))
        return [a for a, pa in enumerate(self.pas) if pa.name not in rigid]

    def evaluate(self):
        p = self.p
        idx = list(range(len(self.pas)))
        P = self.o.solid_program(self._elastic(), idx, eps=p.get('eps', 0.3), alpha=p.get('alpha', 1.0),
                                 beta=p.get('beta', 1.0), eps_xsph=p.get('eps_xsph', 0.5),
                                 grad3d=p.get('grad3d', False))
        self.pairs_last_eval = self.o.solid_group1(P) + self.o.solid_group2(P)
        return self.pairs_last_eval

    def initialise(self):
        if not self._initialised:
            self.evaluate()
            self._initialised = True

    def _stage(self, which, dt):
        for a in self._elastic():
            self.o.stage_solid(a, which, dt)

    def step(self):
        self.initialise()
        self._stage(0, 0.0)
        if self.integrator == 'EPEC':
            self.o.nnps_update()
            self.evaluate()
        self._stage(1, self.dt)
        self.o.update_domain()
        self.o.nnps_update()
        self.evaluate()
        self._stage(2, self.dt)
        self.o.update_domain()
        self.t += self.dt
        self.count += 1
