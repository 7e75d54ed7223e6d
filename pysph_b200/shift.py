"""Particle shifting (pysph/sph/wc/shift.py) on the device: ``SimpleShift``, ``FickianShift``,
``CorrectVelocities`` and the ``ShiftPositions`` tool.

The equations are descriptors (constructor arguments and attributes as in the reference, no
bodies); ``pysph_b200.program`` recognises them, and the reference's own objects, by class name
and turns their Groups into ``('shift', ...)`` / ``('correct_vel', ...)`` ops that run
k_shift / k_correct_velocities (csrc/shift_kernels.cuh).

Deviations from the reference, both documented in DESIGN.md:
  * a Jacobi update: every particle's dpos is formed from the positions before the shift (the
    reference's loop_all moves d_x while later destinations still read s_x);
  * periodic images are formed from the current positions by the wrapping cell grid, where the
    reference's evaluator sees the ghost layer its DomainManager made one stage before.
dpos, gradv and vmax live in device scratch: the tool adds them to the host array, as the
reference does, for name compatibility only; they are not refreshed.
"""
from . import _lib
from .equations import Equation
from .tools import Tool


class SimpleShift(Equation):
    """Xu et al. (2009), eq. 35 (shift.py:41-83):
    dpos_i = beta ri^2 vmax dt sum_j x_ij / (r_ij^3 + 1e-8)"""

    def __init__(self, dest, sources, const=0.04):
        self.beta = const
        super(SimpleShift, self).__init__(dest, sources)


class FickianShift(Equation):
    """Lind et al. (2012), eqs. 21-24 (shift.py:86-148):
    dpos_i = -C h_i |v_i| dt sum_j V_j (1 + f_ij) grad W_ij"""

    def __init__(self, dest, sources, fickian_const=10, tensile_const=0.2,
                 tensile_pow=4, hdx=1.0, tensile_correction=False):
        self.fickian_const = fickian_const
        self.tensile_const = tensile_const
        self.tensile_pow = tensile_pow
        self.hdx = hdx
        self.tensile_correction = tensile_correction
        super(FickianShift, self).__init__(dest, sources)


class CorrectVelocities(Equation):
    """Xu et al. (2009), eq. 34 (shift.py:151-188): u_i += gradv_i . dpos_i, with the
    reference's index order (the transpose of grad v is applied to dpos)"""


_KINDS = {'simple': (_lib.SHIFT_SIMPLE, 0.04), 'fickian': (_lib.SHIFT_FICKIAN, 4)}


class ShiftPositions(Tool):
    """ShiftPositions (shift.py:191-271) on the device.

    Every ``freq``-th step (after steps freq, 2 freq, ...; never with freq = 0) the named
    array's particles are shifted with SimpleShift (shift_kind='simple', constant 0.04) or
    FickianShift ('fickian', constant 4), the constant being ``parameter`` when it is truthy,
    and, with ``correct_velocity``, their velocities corrected with CorrectVelocities.  dt is
    the solver's dt when the tool is made, as in the reference.  Sources are the array's own
    particles: other arrays (walls) are not seen.

    app: anything with ``.solver`` and ``.particles``, or a :class:`B200Solver` itself.

    Nothing is pulled; the host waits for the drift check of each neighbour-search update (one,
    two with the correction).
    """

    def __init__(self, app, array_name, freq=1, shift_kind='simple',
                 correct_velocity=False, parameter=None):
        solver = getattr(app, 'solver', app)
        self.particles = getattr(app, 'particles', None) or solver.particles
        self.dt = solver.dt
        self.dim = int(solver.kernel.dim)
        self.kernel = solver.kernel
        self.freq = freq
        self.kind = shift_kind
        self.correct_velocity = correct_velocity
        self.parameter = parameter
        self.count = 1
        options = ['simple', 'fickian']
        if self.kind not in options:
            raise ValueError('shift_kind should be one of %s' % options)
        arrays = [pa for pa in self.particles if pa.name == array_name]
        be = solver.backend
        if not arrays or array_name not in be.index:
            raise ValueError('ShiftPositions: no particle array %r' % array_name)
        if getattr(solver, 'pm', None) is not None:
            raise NotImplementedError('B200 backend: ShiftPositions with the slab decomposition')
        dom = getattr(solver.nnps, 'domain', None)
        if dom is not None and getattr(dom, 'is_mirror', False):
            raise NotImplementedError('B200 backend: ShiftPositions in a mirror domain')
        self.array = arrays[0]
        kind, default = _KINDS[self.kind]
        self._kind = kind
        self.const = default if not self.parameter else self.parameter
        self._solver = solver
        self._mask = 1 << be.index[array_name]
        # the reference's names on the host array (shift.py:234-253), not refreshed
        arr = self.array
        if 'vmax' not in arr.constants:
            arr.add_constant('vmax', [0.0])
        if 'dpos' not in arr.properties:
            arr.add_property('dpos', stride=3)
        if self.correct_velocity and 'gradv' not in arr.properties:
            arr.add_property('gradv', stride=9)

    def post_step(self, solver):
        if self.freq == 0:
            pass
        elif self.count % self.freq == 0:
            self.shift()
        self.count += 1

    def shift(self):
        """Update the neighbour search, shift; with the correction update it again and correct
        (enqueued)."""
        s = self._solver
        ctx = s.backend.ctx
        s.nnps.update_domain()
        s.nnps.update()
        ctx.call('b200sph_shift', self._mask, self._kind, float(self.dt), float(self.const),
                 1.0, 0, 0.2, 4.0, None)
        if self.correct_velocity:
            s.nnps.update_domain()
            s.nnps.update()
            ctx.call('b200sph_correct_velocities', self._mask, None)
