"""Integrators of the WCSPH hot path on the B200 backend.

Mirrors the reference's integrator interface for this path
(pysph/sph/integrator.py:30-286): construct with ``name=stepper`` keyword
arguments, then ``set_acceleration_evals`` / ``set_nnps`` /
``set_post_stage_callback`` / ``step(t, dt)`` / ``compute_time_step(dt, cfl)``
/ ``initial_acceleration(t, dt)``.  The stage loops the reference generates
from integrator_cython.mako:87-112 are the ``k_stage`` CUDA kernel; the stage
ordering of ``one_timestep`` follows integrator.py:322-420.

Each integrator accepts the steppers it has device kernels for (``steppers``);
another stepper class raises at construction.
"""
from math import sqrt

import numpy as np


class IntegratorStep(object):
    """pysph/sph/integrator_step.py:13-22"""


class WCSPHStep(IntegratorStep):
    """Predictor-corrector stepper: initialize / stage1 / stage2 of
    pysph/sph/integrator_step.py:38-91 (device kernel: k_stage)."""


class WCSPHTVDRK3Step(IntegratorStep):
    """TVD-RK3 stepper: initialize / stage1 / stage2 / stage3 of
    pysph/sph/integrator_step.py:96-168 (device kernel: k_stage_rk3)."""


# stepper class name -> (C-ABI stage call, the same with dt read on the device)
_SUPPORTED_STEPPERS = {
    'WCSPHStep': ('b200sph_stage', 'b200sph_stage_dev'),
    'EDACTVFStep': ('b200sph_stage_tvf', 'b200sph_stage_tvf_dev'),   # wc/edac.py:491-540
    'EDACStep': ('b200sph_stage_edac', 'b200sph_stage_edac_dev'),    # wc/edac.py:82-133
    'SolidMechStep': ('b200sph_stage_solid', 'b200sph_stage_solid_dev'),   # integrator_step.py:173-252
    'WCSPHTVDRK3Step': ('b200sph_stage_rk3', 'b200sph_stage_rk3_dev'),
    'IISPHStep': ('b200sph_stage_iisph', 'b200sph_stage_iisph_dev'),   # iisph.py:22-34
    'GTVFStep': ('b200sph_stage_gtvf', 'b200sph_stage_gtvf_dev'),      # wc/gtvf.py:70-98
    'CRKSPHStep': ('b200sph_stage_crksph', 'b200sph_stage_crksph_dev'),   # wc/crksph.py:884-900
}


class B200Integrator(object):
    # the predictor-corrector steppers (two stages)
    steppers_supported = ('WCSPHStep', 'EDACTVFStep', 'EDACStep', 'SolidMechStep')

    def __init__(self, **kw):
        for name, stepper in kw.items():
            cls = stepper.__class__.__name__
            if cls not in self.steppers_supported:
                raise NotImplementedError(
                    'B200 backend: no device kernel for stepper %r of array %r under '
                    '%s (supported: %s)' % (cls, name, self.__class__.__name__,
                                            self.steppers_supported))
        self.steppers = kw
        self.acceleration_evals = None
        self.nnps = None
        self.parallel_manager = None
        self.fixed_h = False
        self.h_minimum = None
        self.t = 0.0
        self.dt = 0.0
        self._post_stage_callback = None
        self.device_dt = False      # set by B200Solver: dt lives in device memory
        self._stage_arrays = None
        # the adapter is its own "compiled object" (integrator.py:244-247)
        self.c_integrator = self

    # -- wiring (integrator.py:132-144, 214-262) ------------------------------
    def set_acceleration_evals(self, a_evals):
        self.acceleration_evals = list(a_evals)
        backend = self.acceleration_evals[0].backend
        self.backend = backend
        self.ctx = backend.ctx
        missing = [n for n in self.steppers if n not in backend.index]
        if missing:
            raise ValueError('steppers given for unknown arrays %r' % missing)
        kinds = set(s.__class__.__name__ for s in self.steppers.values())
        if set(self.steppers) == set(backend.names) and len(kinds) == 1:
            # one launch for every array
            self._stage_arrays = [(-1,) + _SUPPORTED_STEPPERS[kinds.pop()]]
        else:
            self._stage_arrays = [
                (backend.index[n],) + _SUPPORTED_STEPPERS[s.__class__.__name__]
                for n, s in self.steppers.items()]

    def set_compiled_object(self, c_integrator):
        self.c_integrator = c_integrator

    def set_nnps(self, nnps):
        self.nnps = nnps

    def set_parallel_manager(self, pm):
        self.parallel_manager = pm

    def set_fixed_h(self, fixed_h):
        self.fixed_h = fixed_h

    def set_post_stage_callback(self, callback):
        self._post_stage_callback = callback

    # -- stages ---------------------------------------------------------------
    def _stage(self, which, dt):
        for arr, fn, fn_dev in self._stage_arrays:
            if self.device_dt and which != 0:
                self.ctx.call(fn_dev, arr, which)        # dt read on the device
            else:
                self.ctx.call(fn, arr, which, float(dt))

    def initialize(self):
        self._stage(0, 0.0)

    def stage1(self):
        self._stage(1, self.dt)

    def stage2(self):
        self._stage(2, self.dt)

    def stage3(self):
        self._stage(3, self.dt)

    def do_post_stage(self, stage_dt, stage):
        # integrator_cython.mako:59-74
        if self._post_stage_callback is not None:
            self._post_stage_callback(self.t + stage_dt, self.dt, stage)

    def update_domain(self):
        self.nnps.update_domain()

    def compute_accelerations(self, index=0, update_nnps=True):
        # integrator.py:274-286
        # The decision "are the persistent neighbour lists still valid" (one
        # rank: a drift measurement; several: an all-reduce of it) is enqueued,
        # the evaluation is enqueued behind it on that assumption, and only then
        # does the host wait for the answer -- the GPU never idles on it.  A
        # "no" (once per list lifetime) repeats update + evaluation; everything
        # an evaluation writes is overwritten by the repeat.
        pm = self.parallel_manager
        if update_nnps:
            if pm:
                pm.update(deferred=True)
            self.nnps.update(deferred=True)
        ae = self.acceleration_evals[index]
        ae.device_dt = self.device_dt
        ae.compute(self.t, self.dt)
        if update_nnps:
            redo = pm.confirm() if pm else False
            redo = self.nnps.confirm() or redo
            if redo:
                # (an IISPH evaluation starts the repeat from the pressure the first attempt
                # started from: the library restores it)
                self.nnps.update()
                ae.compute(self.t, self.dt)

    def initial_acceleration(self, t, dt):
        # integrator.py:289-297: evaluate once WITHOUT refreshing the NNPS
        ae = self.acceleration_evals[0]
        ae.device_dt = self.device_dt
        ae.compute(t, dt)

    def step(self, time, dt):
        # integrator_cython.mako:76-82
        self.t = time
        self.dt = dt
        self.one_timestep(time, dt)

    def one_timestep(self, t, dt):
        raise NotImplementedError()

    # -- adaptive time step (integrator.py:146-200) ---------------------------
    def compute_time_step(self, dt, cfl):
        f_cfl, f_force, hmin = self.backend.dt_factors()
        if not self.fixed_h or self.h_minimum is None:
            self.h_minimum = hmin
        hmin = self.h_minimum
        dt_cfl = dt_force = np.inf
        if f_cfl > 0:
            dt_cfl = hmin / f_cfl
        if f_force > 0:
            dt_force = sqrt(hmin / sqrt(f_force))
        dt_min = min(dt_cfl, dt_force)
        if dt_min <= 0.0 or np.isinf(dt_min):
            return None
        return cfl * dt_min


class EulerIntegrator(B200Integrator):
    """integrator.py:312-327.  IISPHStep (iisph.py:22-34) is the only stepper with a device
    stage 1 under it: with any other, stage1 raises."""
    steppers_supported = B200Integrator.steppers_supported + ('IISPHStep',)

    def one_timestep(self, t, dt):   # integrator.py:322-327
        self.compute_accelerations()
        self.stage1()
        self.update_domain()
        self.do_post_stage(dt, 1)

    def stage1(self):
        if any(s.__class__.__name__ != 'IISPHStep' for s in self.steppers.values()):
            raise NotImplementedError(
                'EulerStep has no device kernel on the B200 backend')
        self._stage(1, self.dt)


class PECIntegrator(B200Integrator):
    """Predict - Evaluate - Correct (integrator.py:344-361)."""

    def one_timestep(self, t, dt):
        self.initialize()
        self.stage1()
        self.update_domain()
        self.do_post_stage(0.5 * dt, 1)
        self.compute_accelerations()
        self.stage2()
        self.update_domain()
        self.do_post_stage(dt, 2)


class EPECIntegrator(B200Integrator):
    """Evaluate - Predict - Evaluate - Correct (integrator.py:401-420)."""

    def one_timestep(self, t, dt):
        self.initialize()
        self.compute_accelerations()
        self.stage1()
        self.update_domain()
        self.do_post_stage(0.5 * dt, 1)
        self.compute_accelerations()
        self.stage2()
        self.update_domain()
        self.do_post_stage(dt, 2)


class TVDRK3Integrator(B200Integrator):
    """TVD-RK3 (integrator.py:426-460) with WCSPHTVDRK3Step: three evaluations
    per step; every stage advances by the whole dt from a combination of the
    stage copies and the current state, and the post-stage times are dt/3,
    2dt/3 and dt as in the reference."""
    steppers_supported = ('WCSPHTVDRK3Step',)

    def set_nnps(self, nnps):
        if getattr(getattr(nnps, 'domain', None), 'is_periodic', False):
            # update_domain box-wraps x, y, z but not x0, y0, z0 (nnps_base.pyx:699-743):
            # stages 2 and 3 would combine q0 with a wrapped q and displace a particle
            # that crossed a periodic face by a fraction of the box
            raise NotImplementedError(
                'B200 backend: TVDRK3Integrator in a periodic domain (the periodic wrap '
                'moves x, y, z but not the stage copies x0, y0, z0 that stages 2 and 3 '
                'combine them with)')
        B200Integrator.set_nnps(self, nnps)

    def one_timestep(self, t, dt):
        self.initialize()
        self.compute_accelerations()
        self.stage1()
        self.update_domain()
        self.do_post_stage(1. / 3 * dt, 1)
        self.compute_accelerations()
        self.stage2()
        self.update_domain()
        self.do_post_stage(2. / 3 * dt, 2)
        self.compute_accelerations()
        self.stage3()
        self.update_domain()
        self.do_post_stage(dt, 3)
