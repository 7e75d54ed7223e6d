"""The generalised transport-velocity formulation: PySPH's ``GTVFScheme`` (pysph/sph/wc/gtvf.py,
Zhang, Hu & Adams 2017).

The equation descriptors, ``GTVFStep``, ``GTVFIntegrator`` and the scheme mirror
pysph/sph/wc/gtvf.py.  ``get_equations`` returns a ``MultiStageEquations`` of the reference's
two evaluations (:586-662); ``B200Solver`` gives each its own ``B200AccelerationEval`` and
``pysph_b200.program`` turns each, as a whole, into one ``('gtvf', GtvfProgram, evaluation)``
op: the CUDA passes of ``csrc/gtvf_kernels.cuh``.  ``GTVFStep`` runs under ``GTVFIntegrator``
only (k_stage_gtvf).

Refused with NotImplementedError: several fluid arrays (the reference's CorrectDensity of one
fluid reads another fluid's rho0 before that fluid's own initialize has refreshed it), nu > 0
with walls (SolidWallNoSlipBC reads a V the scheme's fluid arrays do not have), an array whose
asigma is not zero (sigma stays on the host), 1-D, mirror domains, ghost particles and the slab
decomposition.  The solid-mechanics equations of gtvf.py, which the scheme never uses, are not
built.
"""
import numpy as np

from .equations import Equation, Group, MultiStageEquations
from .integrator import B200Integrator, IntegratorStep
from .particle_array import get_particle_array
from .transport_velocity import (ContinuitySolid, MomentumEquationArtificialViscosity,
                                 SetWallVelocity, SolidWallNoSlipBC, SolidWallPressureBC,
                                 StateEquation, VolumeSummation)


class GTVFStep(IntegratorStep):
    """gtvf.py:70-98: a half kick with uhat, the drift with uhat, a half kick (k_stage_gtvf)"""


class GTVFIntegrator(B200Integrator):
    """gtvf.py:52-67: stage1, evaluation 0 without a neighbour-search update, stage2,
    update_domain, evaluation 1, stage3; every post-stage callback gets dt.
    ``initial_acceleration`` (integrator.py:289-297) runs evaluation 0 only, so the first step
    kicks with the au / auhat the arrays were created with."""
    steppers_supported = ('GTVFStep',)

    def one_timestep(self, t, dt):
        self.stage1()
        self.do_post_stage(dt, 1)
        self.compute_accelerations(0, update_nnps=False)
        self.stage2()
        self.update_domain()
        self.do_post_stage(dt, 2)
        self.compute_accelerations(1)
        self.stage3()
        self.do_post_stage(dt, 3)


class ContinuityEquationGTVF(Equation):
    """gtvf.py:101-121"""


class CorrectDensity(Equation):
    """gtvf.py:124-148"""


class MomentumEquationPressureGradient(Equation):
    """gtvf.py:151-250 (recognised by its module: the EDAC and transport-velocity equations of
    this name are others)"""

    def __init__(self, dest, sources, pref, gx=0.0, gy=0.0, gz=0.0):
        self.pref = pref
        self.gx = gx
        self.gy = gy
        self.gz = gz
        super(MomentumEquationPressureGradient, self).__init__(dest, sources)


class MomentumEquationViscosity(Equation):
    """gtvf.py:253-288"""

    def __init__(self, dest, sources, nu):
        self.nu = nu
        super(MomentumEquationViscosity, self).__init__(dest, sources)


class MomentumEquationArtificialStress(Equation):
    """gtvf.py:291-348"""

    def __init__(self, dest, sources, dim):
        self.dim = dim
        super(MomentumEquationArtificialStress, self).__init__(dest, sources)


GTVF_PROPS = ('uhat', 'vhat', 'what', 'rho0', 'rhodiv', 'p0', 'auhat', 'avhat', 'awhat', 'arho',
              'arho0')
GTVF_STRIDED = ('gradvhat', 'sigma', 'asigma')
GTVF_OUTPUT = ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'p', 'h', 'm', 'au', 'av', 'aw', 'pid', 'gid',
               'tag']
SOLID_PROPS = ('uf', 'vf', 'wf', 'vg', 'ug', 'wij', 'wg', 'V')


def get_particle_array_gtvf(constants=None, **props):
    """gtvf.py:32-49"""
    pa = get_particle_array(additional_props=GTVF_PROPS, constants=constants, **props)
    for name in GTVF_STRIDED:
        pa.add_property(name, stride=9)
    pa.set_output_arrays(GTVF_OUTPUT)
    return pa


class GTVFScheme(object):
    def __init__(self, fluids, solids, dim, rho0, c0, nu, h0, pref, gx=0.0, gy=0.0, gz=0.0,
                 b=1.0, alpha=0.0):
        self.fluids = fluids
        self.solids = solids
        self.dim = dim
        self.rho0 = rho0
        self.c0 = c0
        self.nu = nu
        self.h0 = h0
        self.pref = pref
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.b = b
        self.alpha = alpha
        self.solver = None

    def configure(self, **kw):                          # scheme.py: Scheme.configure
        for k, v in kw.items():
            if not hasattr(self, k):
                raise RuntimeError('Parameter {param} not defined for {scheme}.'
                                   .format(param=k, scheme=self.__class__.__name__))
            setattr(self, k, v)

    def get_steppers(self):                             # configure_solver, gtvf.py:565-572
        return dict((f, GTVFStep()) for f in self.fluids)

    def get_equations(self):                            # gtvf.py:586-662
        all_ = self.fluids + self.solids
        stage1 = []
        if self.solids:
            stage1.append(Group(equations=[SetWallVelocity(dest=s, sources=self.fluids)
                                           for s in self.solids], real=False))
        eq1 = []
        for fluid in self.fluids:
            eq1.append(ContinuityEquationGTVF(dest=fluid, sources=self.fluids))
            if self.solids:
                eq1.append(ContinuitySolid(dest=fluid, sources=self.solids))
        stage1.append(Group(equations=eq1, real=False))

        stage2 = [Group(equations=[CorrectDensity(dest=f, sources=all_) for f in self.fluids],
                        real=False),
                  Group(equations=[StateEquation(dest=f, sources=None, p0=self.pref,
                                                 rho0=self.rho0, b=1.0) for f in self.fluids],
                        real=False)]
        g2_s = []
        for solid in self.solids:
            g2_s.append(VolumeSummation(dest=solid, sources=all_))
            g2_s.append(SolidWallPressureBC(dest=solid, sources=self.fluids, b=1.0, rho0=self.rho0,
                                            p0=self.pref, gx=self.gx, gy=self.gy, gz=self.gz))
        if g2_s:
            stage2.append(Group(equations=g2_s, real=False))
        eq4 = []
        for fluid in self.fluids:
            eq4.append(MomentumEquationPressureGradient(dest=fluid, sources=all_, pref=self.pref,
                                                        gx=self.gx, gy=self.gy, gz=self.gz))
            if self.alpha > 0.0:
                eq4.append(MomentumEquationArtificialViscosity(dest=fluid, sources=all_,
                                                               c0=self.c0, alpha=self.alpha))
            if self.nu > 0.0:
                eq4.append(MomentumEquationViscosity(dest=fluid, sources=all_, nu=self.nu))
                if self.solids:
                    eq4.append(SolidWallNoSlipBC(dest=fluid, sources=self.solids, nu=self.nu))
            eq4.append(MomentumEquationArtificialStress(dest=fluid, sources=self.fluids,
                                                        dim=self.dim))
        stage2.append(Group(equations=eq4, real=True))
        return MultiStageEquations([stage1, stage2])

    def setup_properties(self, particles, clean=True):  # gtvf.py:664-680
        by_name = dict((p.name, p) for p in particles)
        for name in self.fluids + self.solids:
            pa = by_name[name]
            want = GTVF_PROPS + (SOLID_PROPS if name in self.solids else ())
            for p in want:
                if p not in pa.properties:
                    pa.add_property(p)
            for p in GTVF_STRIDED:
                if p not in pa.properties:
                    pa.add_property(p, stride=9)
            pa.set_output_arrays(GTVF_OUTPUT)


def make_gtvf_solver(particles, scheme, kernel, dt, domain=None, device=0, **solver_kw):
    """A solver for a :class:`GTVFScheme` as its configure_solver makes it (gtvf.py:545-584):
    GTVFIntegrator with GTVFStep for every fluid.  The arrays carry no dt_cfl / dt_force, so
    adaptive_timestep=True keeps dt fixed, as in the reference."""
    from .solver import B200Solver
    for pa in particles:
        if 'asigma' in pa.properties and np.any(pa.properties['asigma'] != 0.0):
            raise NotImplementedError(
                'B200 backend: GTVF array %r has a non-zero asigma (sigma and asigma stay on the '
                'host; GTVFScheme writes neither)' % pa.name)
    integ = GTVFIntegrator(**scheme.get_steppers())
    kw = dict(adaptive_timestep=False, tf=1e9, fixed_h=True, device=device, domain=domain)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integ, dt=dt, **kw)
