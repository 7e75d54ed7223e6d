"""Implicit incompressible SPH: PySPH's ``IISPHScheme`` (pysph/sph/iisph.py, Ihmsen et al. 2014).

The equation descriptors, ``IISPHStep`` and the scheme mirror pysph/sph/iisph.py; ``get_equations``
emits the reference's Groups in the reference's order (:511-643), and ``pysph_b200.program``
turns those Groups, as a whole, into one ``('iisph', IisphProgram)`` op: the CUDA passes of
``csrc/iisph_kernels.cuh`` with the pressure iterations decided on the device.  ``IISPHStep``
runs under ``EulerIntegrator`` (k_stage_iisph).

Deviation: ``debug=True`` is accepted but prints nothing per iteration (the host never sees the
iterations; ``pysph_b200.iisph.last_iterations`` reads the last evaluation's count).
"""
import ctypes as C

import numpy as np

from .equations import Equation, Group
from .integrator import IntegratorStep
from .particle_array import get_particle_array


class IISPHStep(IntegratorStep):
    """iisph.py:22-34: u = uadv + dt au, x += dt u (device kernel: k_stage_iisph)"""


class NumberDensity(Equation):
    """iisph.py:37-42"""


class SummationDensity(Equation):
    """iisph.py:45-50 (recognised by its module: not basic_equations' SummationDensity)"""


class SummationDensityBoundary(Equation):
    """iisph.py:53-59"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(SummationDensityBoundary, self).__init__(dest, sources)


class AdvectionAcceleration(Equation):
    """iisph.py:79-98"""

    def __init__(self, dest, sources, gx=0.0, gy=0.0, gz=0.0):
        self.gx, self.gy, self.gz = gx, gy, gz
        super(AdvectionAcceleration, self).__init__(dest, sources)


class ViscosityAcceleration(Equation):
    """iisph.py:101-112"""

    def __init__(self, dest, sources, nu):
        self.nu = nu
        super(ViscosityAcceleration, self).__init__(dest, sources)


class ViscosityAccelerationBoundary(Equation):
    """iisph.py:115-131"""

    def __init__(self, dest, sources, rho0, nu):
        self.nu = nu
        self.rho0 = rho0
        super(ViscosityAccelerationBoundary, self).__init__(dest, sources)


class ComputeDII(Equation):
    """iisph.py:134-146"""


class ComputeDIIBoundary(Equation):
    """iisph.py:149-160"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(ComputeDIIBoundary, self).__init__(dest, sources)


class ComputeRhoAdvection(Equation):
    """iisph.py:163-176"""


class ComputeRhoBoundary(Equation):
    """iisph.py:179-191"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(ComputeRhoBoundary, self).__init__(dest, sources)


class ComputeAII(Equation):
    """iisph.py:194-207"""


class ComputeAIIBoundary(Equation):
    """iisph.py:210-225"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(ComputeAIIBoundary, self).__init__(dest, sources)


class ComputeDIJPJ(Equation):
    """iisph.py:228-240"""


class UpdateGhostProps(Equation):
    """iisph.py:243-261 (copies to ghost particles: the device's periodic grid has none)"""

    def __init__(self, dest, sources=None):
        super(UpdateGhostProps, self).__init__(dest, sources)


class PressureSolve(Equation):
    """iisph.py:264-341.  The iterations and their convergence test run on the device, so
    ``compression`` / ``converged()`` are not updated on the host."""

    def __init__(self, dest, sources, rho0, omega=0.5, tolerance=1e-2, debug=False):
        self.rho0 = rho0
        self.omega = omega
        self.compression = 0.0
        self.debug = debug
        self.tolerance = tolerance
        super(PressureSolve, self).__init__(dest, sources)


class PressureSolveBoundary(Equation):
    """iisph.py:344-355"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(PressureSolveBoundary, self).__init__(dest, sources)


class UpdateGhostPressure(Equation):
    """iisph.py:358-364 (copies to ghost particles: none on the device)"""


class PressureForce(Equation):
    """iisph.py:367-389"""


class PressureForceBoundary(Equation):
    """iisph.py:392-402"""

    def __init__(self, dest, sources, rho0):
        self.rho0 = rho0
        super(PressureForceBoundary, self).__init__(dest, sources)


# pysph/base/utils.py:226-230
IISPH_PROPS = ('uadv', 'vadv', 'wadv', 'rho_adv', 'au', 'av', 'aw', 'ax', 'ay', 'az',
               'dii0', 'dii1', 'dii2', 'V', 'dt_cfl', 'dt_force', 'aii', 'dijpj0', 'dijpj1',
               'dijpj2', 'p', 'p0', 'piter', 'compression')


def get_particle_array_iisph(constants=None, **props):
    """pysph/base/utils.py:193-236: the property set of IISPHScheme's arrays (fluids and
    solids alike), the constant tmp_comp and the reference's output arrays."""
    consts = {'tmp_comp': [0.0, 0.0]}
    if constants:
        consts.update(constants)
    pa = get_particle_array(additional_props=IISPH_PROPS, constants=consts, **props)
    pa.set_output_arrays(['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'h', 'm', 'p', 'pid', 'au',
                          'av', 'aw', 'tag', 'gid', 'V'])
    return pa


class IISPHScheme(object):
    def __init__(self, fluids, solids, dim, rho0, nu=0.0, gx=0.0, gy=0.0, gz=0.0, omega=0.5,
                 tolerance=1e-2, debug=False, has_ghosts=False):
        self.fluids = fluids
        self.solids = solids
        self.dim = dim
        self.rho0 = rho0
        self.nu = nu
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.omega = omega
        self.tolerance = tolerance
        self.debug = debug
        self.has_ghosts = has_ghosts

    def configure(self, **kw):                          # scheme.py: Scheme.configure
        for k, v in kw.items():
            if not hasattr(self, k):
                raise RuntimeError('Parameter {param} not defined for {scheme}.'
                                   .format(param=k, scheme=self.__class__.__name__))
            setattr(self, k, v)

    def get_steppers(self):                             # configure_solver, :496-505
        return dict((f, IISPHStep()) for f in self.fluids)

    def get_equations(self):                            # iisph.py:511-643
        equations = []
        if self.solids:
            equations.append(Group(equations=[NumberDensity(dest=x, sources=[x])
                                              for x in self.solids]))
        equations.append(Group(equations=[SummationDensity(dest=x, sources=self.fluids)
                                          for x in self.fluids], real=False))
        if self.solids:
            equations.append(Group(equations=[
                SummationDensityBoundary(dest=x, sources=self.solids, rho0=self.rho0)
                for x in self.fluids], real=False))
        eq = []
        for fluid in self.fluids:
            eq.extend([AdvectionAcceleration(dest=fluid, sources=None, gx=self.gx, gy=self.gy,
                                             gz=self.gz),
                       ComputeDII(dest=fluid, sources=self.fluids)])
            if self.nu > 0.0:
                eq.append(ViscosityAcceleration(dest=fluid, sources=self.fluids, nu=self.nu))
            if self.solids:
                if self.nu > 0.0:
                    eq.append(ViscosityAccelerationBoundary(dest=fluid, sources=self.solids,
                                                            nu=self.nu, rho0=self.rho0))
                eq.append(ComputeDIIBoundary(dest=fluid, sources=self.solids, rho0=self.rho0))
        equations.append(Group(equations=eq, real=False))
        eq = []
        for fluid in self.fluids:
            eq.extend([ComputeRhoAdvection(dest=fluid, sources=self.fluids),
                       ComputeAII(dest=fluid, sources=self.fluids)])
            if self.solids:
                eq.extend([ComputeRhoBoundary(dest=fluid, sources=self.solids, rho0=self.rho0),
                           ComputeAIIBoundary(dest=fluid, sources=self.solids, rho0=self.rho0)])
        equations.append(Group(equations=eq))
        sg1 = Group(equations=[ComputeDIJPJ(dest=x, sources=self.fluids) for x in self.fluids])
        eq = []
        for fluid in self.fluids:
            eq.append(PressureSolve(dest=fluid, sources=self.fluids, rho0=self.rho0,
                                    tolerance=self.tolerance, debug=self.debug))
            if self.solids:
                eq.append(PressureSolveBoundary(dest=fluid, sources=self.solids, rho0=self.rho0))
        sg2 = Group(equations=eq)
        if self.has_ghosts:
            ghost1 = Group(equations=[UpdateGhostProps(dest=x, sources=None) for x in self.fluids],
                           real=False)
            ghost2 = Group(equations=[UpdateGhostPressure(dest=x, sources=None)
                                      for x in self.fluids], real=False)
            solver_eqs = [sg1, ghost1, sg2, ghost2]
        else:
            solver_eqs = [sg1, sg2]
        equations.append(Group(equations=solver_eqs, iterate=True, max_iterations=30,
                               min_iterations=2))
        eq = []
        for fluid in self.fluids:
            eq.append(PressureForce(dest=fluid, sources=self.fluids))
            if self.solids:
                eq.append(PressureForceBoundary(dest=fluid, sources=self.solids, rho0=self.rho0))
        equations.append(Group(equations=eq))
        return equations

    def setup_properties(self, particles, clean=True):  # iisph.py:645-672
        dummy = get_particle_array_iisph()
        for pa in particles:
            for name in dummy.properties:
                if name not in pa.properties:
                    pa.add_property(name)
            for c, v in dummy.constants.items():
                if c not in pa.constants:
                    pa.add_constant(c, v)
            pa.set_output_arrays(dummy.output_property_arrays)


def last_iterations(solver_or_eval):
    """(iterations, {fluid name: compression}) of the last IISPH evaluation, read back from the
    device (waits for it)."""
    ae = getattr(solver_or_eval, 'a_eval', solver_or_eval)
    it = C.c_int(0)
    comp = (C.c_double * 8)()
    ae.ctx.call('b200sph_iisph_stats', C.byref(it), comp)
    fluids = getattr(ae, 'iisph_fluids', ())
    return it.value, dict((ae.backend.names[i], comp[i]) for i in fluids)


def make_iisph_solver(particles, scheme, kernel, dt, domain=None, device=0, **solver_kw):
    """A solver for an :class:`IISPHScheme` as its configure_solver makes it (iisph.py:469-509):
    EulerIntegrator with IISPHStep for every fluid.  dt is the initial step; pass
    adaptive_timestep=True (and cfl) as dam_break_2d.py does for its adaptive IISPH run."""
    from .integrator import EulerIntegrator
    from .solver import B200Solver
    integ = EulerIntegrator(**scheme.get_steppers())
    kw = dict(adaptive_timestep=False, tf=1e9, fixed_h=True, device=device, domain=domain)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integ, dt=dt, **kw)
