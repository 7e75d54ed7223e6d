"""Solver tools (pysph/solver/tools.py): ``DensityCorrection``.

A tool is an object with ``pre_step(solver)``, ``post_stage(t, dt, stage)`` and / or
``post_step(solver)`` methods; ``B200Solver.add_tool`` registers the ones a tool overloads,
as ``Application.add_tool`` does (application.py:1358-1369, :1470-1475).
"""
from . import _lib
from .kernels import kernel_id


class Tool(object):
    """pysph/solver/tools.py:6-36: overload any of these."""

    def pre_step(self, solver):
        pass

    def post_stage(self, current_time, dt, stage):
        pass

    def post_step(self, solver):
        pass


def is_overloaded_method(obj, name):
    """True when the class of ``obj`` defines ``name`` itself rather than inheriting it from
    a base class called Tool (this module's or the reference's)."""
    for klass in type(obj).__mro__:
        if name in vars(klass):
            return klass.__name__ != 'Tool'
    return False


_CORR = {'shepard': _lib.DFILTER_SHEPARD, 'mls2d_1': _lib.DFILTER_MLS2D,
         'mls3d_1': _lib.DFILTER_MLS3D}
_CORR_DIM = {'mls2d_1': 2, 'mls3d_1': 3}


class DensityCorrection(Tool):
    """Periodic density re-initialisation (pysph/solver/tools.py:97-205) on the device.

    Every ``freq``-th step (after steps freq, 2 freq, ...; never with freq = 0) the density of
    each array named in ``arr_names`` is re-initialised from the array's own particles with
    ShepardFilter (corr='shepard'), MLSFirstOrder2D ('mls2d_1') or MLSFirstOrder3D ('mls3d_1'),
    smoothed with ``kernel`` (a kernel class; None: the solver's).  Like the reference's
    evaluator, it first updates the neighbour search for the current positions.

    app: anything with ``.solver`` and ``.particles``, or a :class:`B200Solver` itself.

    The tool reads neither t nor dt and pulls nothing; its one host wait per filter call is
    the drift check of that neighbour-search update.
    """

    def __init__(self, app, arr_names, corr='shepard', freq=10, kernel=None):
        solver = getattr(app, 'solver', app)
        particles = getattr(app, 'particles', None) or solver.particles
        if corr not in _CORR:
            raise ValueError('corr should be one of %s' % list(_CORR))
        self.freq = freq
        self.corr = corr
        self.names = list(arr_names)
        self.count = 1
        self.particles = particles
        self.dim = int(solver.kernel.dim)
        kcls = kernel if kernel is not None else solver.kernel.__class__
        self.kernel = kcls(dim=self.dim)
        if corr in _CORR_DIM and self.dim != _CORR_DIM[corr]:
            raise NotImplementedError('B200 backend: DensityCorrection(corr=%r) needs dim = %d, '
                                      'the solver has dim = %d' % (corr, _CORR_DIM[corr], self.dim))
        if getattr(solver, 'pm', None) is not None:
            raise NotImplementedError('B200 backend: DensityCorrection with the slab decomposition')
        dom = getattr(solver.nnps, 'domain', None)
        if dom is not None and (getattr(dom, 'is_periodic', False) or getattr(dom, 'is_mirror', False)):
            raise NotImplementedError('B200 backend: DensityCorrection in a periodic or mirror domain')
        if self.kernel.radius_scale > solver.kernel.radius_scale:
            raise NotImplementedError(
                'B200 backend: DensityCorrection(kernel=%s) reaches further (radius scale %g) than '
                'the solver\'s %s, which the neighbour lists are built for'
                % (kcls.__name__, self.kernel.radius_scale, solver.kernel.__class__.__name__))
        be = solver.backend
        for name in self.names:
            if name not in be.index:
                raise ValueError('DensityCorrection: no particle array %r' % name)
        self._solver = solver
        self._kid = kernel_id(self.kernel)
        self._mask = sum(1 << be.index[n] for n in self.names)
        # rhotmp, as the reference adds it (tools.py:142): on the host arrays and on the device
        for pa in self.particles:
            if pa.name in self.names and 'rhotmp' not in pa.properties:
                pa.add_property('rhotmp')
        self._rhotmp = be.add_user_property('rhotmp')

    def post_step(self, solver):
        if self.freq == 0:
            pass
        elif self.count % self.freq == 0:
            self.filter()
        self.count += 1

    def filter(self):
        """Update the neighbour search for the current positions, then filter (enqueued)."""
        s = self._solver
        s.nnps.update_domain()
        s.nnps.update()
        s.backend.ctx.call('b200sph_density_filter', self._mask, _CORR[self.corr], self._kid,
                           self._rhotmp, 0)
