"""PySPH's Interpolator (pysph/tools/interpolator.py:175-510) on the device.

``Interpolator`` evaluates a particle property at arbitrary points -- a uniform grid over the
particles by default -- with the reference's five methods ('shepard', 'sph', 'splash',
'splash_norm', 'order1'), its signatures, attributes and result shapes.  The points live on the
device (``b200sph_probe_create``); each ``interpolate`` is one ``b200sph_interpolate`` call.

Two modes, chosen from the arrays themselves:

* live: every array is bound (``pa.gpu``) to the :class:`B200Backend` of a running solver.  The
  call reads that context's current device state -- positions, h, m, rho and the property --
  and changes nothing the solver caches: the run is bitwise the same with or without probes.
* private: host arrays, e.g. from :func:`pysph_b200.load` or the reference's ``iter_output``.
  The Interpolator owns a backend and a :class:`B200NNPS` built for its kernel and
  ``domain_manager``; ``update_particle_arrays`` pushes new arrays, ``update`` re-pushes the same
  arrays after their particles moved.  As in the reference, ``interpolate`` reads the property's
  current host values on every call.

Deviations from the reference (DESIGN.md, "Interpolator"): ``equations`` other than None raise
NotImplementedError, and 'order1' never overwrites the arrays' ``rho`` (the reference's
SummationDensity Group does, as a side effect).
"""
import ctypes as C

import numpy as np

from . import _lib
from .backend import B200Backend, B200DeviceHelper, _host_array
from .kernels import Gaussian, kernel_id
from .nnps import B200NNPS


def get_bounding_box(particle_arrays, tight=False, stretch=0.05):
    """Find the size of the domain given a sequence of particle arrays.

    If `tight` is True, the bounds are tight, if not the domain is stretched
    along each dimension by an amount `stretch` specified as a percentage of
    the length along that dimension is added in each dimension.
    """
    xmin, xmax = 1e20, -1e20
    ymin, ymax = 1e20, -1e20
    zmin, zmax = 1e20, -1e20
    for pa in particle_arrays:
        x, y, z = pa.x, pa.y, pa.z
        xmin = min(xmin, x.min())
        xmax = max(xmax, x.max())
        ymin = min(ymin, y.min())
        ymax = max(ymax, y.max())
        zmin = min(zmin, z.min())
        zmax = max(zmax, z.max())

    bounds = np.asarray((xmin, xmax, ymin, ymax, zmin, zmax))
    if not tight:
        lengths = stretch * np.repeat(bounds[1::2] - bounds[::2], 2)
        lengths[::2] *= -1.0
        bounds += lengths
    return bounds


def get_nx_ny_nz(num_points, bounds):
    """Given a number of points to use and the bounds, return a triplet
    of integers for a uniform mesh with approximately that many points.
    """
    bounds = np.asarray(bounds, dtype=float)
    length = bounds[1::2] - bounds[::2]
    total_length = length.sum()
    rel_length = length / total_length
    non_zero = rel_length > 1e-3
    dim = int(non_zero.sum())
    volume = np.prod(length[non_zero])
    delta = pow(volume / num_points, 1.0 / dim)
    dimensions = np.ones(3, dtype=int)
    for i in range(3):
        if rel_length[i] > 1e-4:
            dimensions[i] = int(round(length[i] / delta))
    return dimensions


class Interpolator(object):
    """Interpolate particle properties onto a uniform grid or a given set of points."""

    METHODS = ['shepard', 'sph', 'order1', 'splash', 'splash_norm']

    def __init__(self, particle_arrays, num_points=125000, kernel=None,
                 x=None, y=None, z=None, domain_manager=None,
                 equations=None, method='shepard'):
        if equations is not None:
            raise NotImplementedError('B200 backend: Interpolator(equations=...): only the '
                                      'built-in methods %s run on the device' % self.METHODS)
        self._backend = self._nnps = None
        self._probe = None
        self._private = False
        self.domain_manager = domain_manager
        self.equations = None
        self.method = method
        self._set_particle_arrays(particle_arrays)
        bounds = get_bounding_box(self.particle_arrays)
        shape = get_nx_ny_nz(num_points, bounds)
        self.dim = 3 - list(shape).count(1)
        self.kernel = Gaussian(dim=self.dim) if kernel is None else kernel
        self._kid = kernel_id(self.kernel)
        if method not in self.METHODS:
            raise RuntimeError('%s method is not implemented' % (method))
        if method == 'order1' and int(self.kernel.dim) != self.dim:
            raise NotImplementedError('B200 backend: order1 with a %d-D kernel for %d-D data'
                                      % (self.kernel.dim, self.dim))
        self._bind(self.particle_arrays)
        if x is None and y is None and z is None:
            self.set_domain(bounds, shape)
        else:
            self.set_interpolation_points(x=x, y=y, z=z)

    # ## Interpolator protocol ###############################################
    def set_interpolation_points(self, x=None, y=None, z=None):
        """Set the points on which we must interpolate the arrays.

        If any of x, y, z is not passed it is assumed to be 0.0 and shaped
        like the other non-None arrays.
        """
        tmp = None
        for tmp in (x, y, z):
            if tmp is not None:
                break
        if tmp is None:
            raise RuntimeError('At least one non-None array must be given.')

        def _get_array(_t):
            return np.asarray(_t) if _t is not None else np.zeros_like(tmp)

        x, y, z = _get_array(x), _get_array(y), _get_array(z)
        self.shape = x.shape
        self.x, self.y, self.z = x.squeeze(), y.squeeze(), z.squeeze()
        self._points = [np.ascontiguousarray(c.ravel(), dtype=np.float64) for c in (x, y, z)]
        self._hp = self._get_max_h_in_arrays()
        self._make_probe()

    def set_domain(self, bounds, shape):
        """Set the domain to interpolate into: bounds (xmin, xmax, ymin, ymax, zmin, zmax),
        shape (nx, ny, nz)."""
        self.bounds = np.asarray(bounds)
        self.shape = np.asarray(shape)
        x, y, z = self._create_default_points(self.bounds, self.shape)
        self.set_interpolation_points(x, y, z)

    def interpolate(self, prop, comp=0):
        """Interpolate the property `prop`; with 'order1', `comp` 1, 2, 3 selects a component
        of its gradient.  Returns an array shaped like the points."""
        assert isinstance(comp, int), 'Error: only interger value is allowed'
        single = self.method in ['sph', 'shepard', 'splash', 'splash_norm']
        if comp and single:
            raise RuntimeError("Error: use 'order1' method to evaluate"
                               "gradient")
        if not single and comp > 3:
            raise RuntimeError("Error: Only 0, 1, 2, 3 allowed")
        props = (C.c_int * _lib.MAX_ARRAYS)(*([-1] * _lib.MAX_ARRAYS))
        for i, pa in zip(self._index, self.particle_arrays):
            props[i] = self._prop_id(i, pa, prop)
        n = len(self._points[0])
        out = np.zeros(n * (1 if single else 4), dtype=np.float64)
        self._backend.ctx.call('b200sph_interpolate', self._probe, _lib.INTERP_METHODS[self.method],
                               self._kid, int(self.kernel.dim), props, self._mask, out.ctypes.data)
        result = out if single else out[comp::4].copy()
        result.shape = self.shape
        return result.squeeze()

    def update(self, update_domain=True):
        """Update the neighbour search when particles have moved (private mode: the arrays'
        host values are pushed again).  Live, the solver keeps its own search current and
        every ``interpolate`` sees the device state: nothing to do."""
        if not self._private:
            return
        self._backend.push_all()
        if update_domain:
            self._nnps.update_domain()
        self._nnps.update()

    def update_particle_arrays(self, particle_arrays):
        """Call this for a new set of particle arrays which have the same properties as
        before, e.g. each time a new output file is loaded."""
        self._set_particle_arrays(particle_arrays)
        self._bind(self.particle_arrays)
        self._make_probe()

    # ### Private protocol ###################################################
    def _bind(self, arrays):
        """Live when every array is bound to one solver's backend, else a private backend."""
        self._release_probe()
        helpers = [getattr(pa, 'gpu', None) for pa in arrays]
        bound = [isinstance(g, B200DeviceHelper) for g in helpers]
        if all(bound):
            if len(set(id(g._backend) for g in helpers)) != 1:
                raise ValueError('Interpolator: the arrays are bound to different backends')
            self._backend, self._nnps, self._private = helpers[0]._backend, None, False
            self._index = [g._index for g in helpers]
            self._mask = sum(1 << i for i in self._index)
            return
        if any(bound):
            raise ValueError('Interpolator: some arrays are bound to a device backend and some '
                             'are not; pass the arrays of one running solver or host arrays only')
        if self._private and self._backend.names == [pa.name for pa in arrays]:
            # the same arrays, new data: push (resizing where the counts changed), rebuild
            self._backend.particle_arrays = list(arrays)
            self._unbound(arrays, self._backend.push_all)
            self._nnps.update_domain()
            self._nnps.update()
        else:
            be = self._unbound(arrays, lambda: B200Backend(arrays))
            self._temp = be.add_user_property('temp_prop')
            self._backend, self._private = be, True
            self._nnps = B200NNPS(self.kernel.dim, arrays, backend=be, kernel=self.kernel,
                                  domain=self.domain_manager)
        self._index = list(range(len(arrays)))
        self._mask = (1 << len(arrays)) - 1

    @staticmethod
    def _unbound(arrays, fn):
        """fn() with the arrays' ``gpu`` attribute restored afterwards: a private backend
        does not bind the caller's host arrays."""
        saved = [getattr(pa, 'gpu', None) for pa in arrays]
        try:
            return fn()
        finally:
            for pa, g in zip(arrays, saved):
                pa.gpu = g

    def _prop_id(self, i, pa, prop):
        if prop not in pa.properties:
            return -1
        if self._private:
            n = pa.get_number_of_particles()
            a = np.ascontiguousarray(_host_array(pa, prop), dtype=np.float64)
            if a.size != n:
                raise ValueError('Interpolator: %s.%s has %d values for %d particles'
                                 % (pa.name, prop, a.size, n))
            self._backend.ctx.call('b200sph_push_f64', i, self._temp, a.ctypes.data, 0, n)
            return self._temp
        pid = self._backend.prop_ids[i].get(prop)
        if pid is None:
            raise NotImplementedError('B200 backend: %s.%s is not on the device; a live '
                                      'Interpolator reads device properties only' % (pa.name, prop))
        return pid

    def _make_probe(self):
        if getattr(self, '_points', None) is None:
            return
        self._release_probe()
        x, y, z = self._points
        self._probe = self._backend.ctx.call('b200sph_probe_create', len(x), x.ctypes.data,
                                             y.ctypes.data, z.ctypes.data, float(self._hp))

    def _release_probe(self):
        if self._probe is not None and self._backend is not None:
            self._backend.ctx.call('b200sph_probe_release', self._probe)
        self._probe = None

    def __del__(self):
        try:
            self._release_probe()
        except Exception:
            pass

    def _create_default_points(self, bounds, shape):
        b = bounds
        n = shape
        x, y, z = np.mgrid[
            b[0]:b[1]:n[0] * 1j,
            b[2]:b[3]:n[1] * 1j,
            b[4]:b[5]:n[2] * 1j,
        ]
        return x, y, z

    def _get_max_h_in_arrays(self):
        hmax = -1.0
        for array in self.particle_arrays:
            hmax = max(array.h.max(), hmax)
        return hmax

    def _set_particle_arrays(self, particle_arrays):
        self.particle_arrays = list(particle_arrays)
