"""Conservative reproducing-kernel SPH: PySPH's ``CRKSPHScheme`` (pysph/sph/wc/crksph.py,
Frontiere, Raskin & Owen 2017).

The equation descriptors, ``CRKSPHStep``, ``CRKSPHIntegrator`` and the scheme mirror
pysph/sph/wc/crksph.py.  ``get_equations`` returns a ``MultiStageEquations`` of the reference's
two evaluations (:978-1127); ``B200Solver`` gives each its own ``B200AccelerationEval`` and
``pysph_b200.program`` turns each, as a whole, into one ``('crksph', CrksphProgram, evaluation)``
op: the CUDA passes of ``csrc/crksph_kernels.cuh``.  ``CRKSPHStep`` runs under
``CRKSPHIntegrator`` only (k_stage_crksph).

Properties: p in the fp64 pressure slot, e, ae, cs, V, ai, au .. aw and the strided bi, gradai,
gradbi and gradv in the scheme's fp64 group (one device id per component).  A strided property is
indexed with stride dim, not with the stride it was allocated with (in 2-D, bi holds 2 i + a and
gradbi 4 i + 2 g + a at the front of its buffer), and push / pull keep that layout.  cwij and
rhofac, which the reference leaves at the last pair's value and the density's denominator, stay on
the host.

Refused with NotImplementedError or a library error: several fluid arrays (the reference's
CRKSPHPreStep.loop_all keeps only the last source's moments), ghost particles (has_ghosts=True
with materialised ghosts; a periodic box runs through DomainManager), mirror domains, the slab
decomposition and 1-D.
"""
from .equations import Equation, Group, LaminarViscosity, MultiStageEquations
from .integrator import B200Integrator, IntegratorStep
from .particle_array import get_particle_array


class CRKSPHStep(IntegratorStep):
    """crksph.py:884-900: u0 = u | u += dt au | e += dt ae, x += dt/2 (u + u0) (k_stage_crksph)"""


class CRKSPHIntegrator(B200Integrator):
    """crksph.py:866-881: stage1, evaluation 0, stage2, evaluation 1, stage3, update_domain;
    both evaluations update the neighbour search, and every post-stage callback gets dt.
    ``initial_acceleration`` (integrator.py:289-297) runs evaluation 0."""
    steppers_supported = ('CRKSPHStep',)

    def one_timestep(self, t, dt):
        self.stage1()
        self.do_post_stage(dt, 1)
        self.compute_accelerations(0)
        self.stage2()
        self.do_post_stage(dt, 2)
        self.compute_accelerations(1)
        self.stage3()
        self.do_post_stage(dt, 3)
        self.update_domain()


class CRKSPHPreStep(Equation):
    """crksph.py:32-167"""

    def __init__(self, dest, sources, dim=2):
        self.dim = dim
        super(CRKSPHPreStep, self).__init__(dest, sources)


class CRKSPHSymmetric(Equation):
    """crksph.py:280-388"""

    def __init__(self, dest, sources, dim=2, tol=0.5):
        self.dim = dim
        self.tol = tol
        super(CRKSPHSymmetric, self).__init__(dest, sources)


class NumberDensity(Equation):
    """crksph.py:391-406"""


class SummationDensityCRKSPH(Equation):
    """crksph.py:409-441"""


class VelocityGradient(Equation):
    """crksph.py:444-477"""

    def __init__(self, dest, sources, dim):
        self.dim = dim
        super(VelocityGradient, self).__init__(dest, sources)


class MomentumEquation(Equation):
    """crksph.py:480-632 (recognised by its module: the WCSPH equation of this name is another)"""

    def __init__(self, dest, sources, dim, gx=0.0, gy=0.0, gz=0.0, cl=2, cq=1, eta_crit=0.3,
                 eta_fold=0.2, tol=0.5):
        self.dim = dim
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.cl = cl
        self.cq = cq
        self.eta_crit = eta_crit
        self.eta_fold = eta_fold
        self.tol = tol
        super(MomentumEquation, self).__init__(dest, sources)


class EnergyEquation(Equation):
    """crksph.py:635-783"""

    def __init__(self, dest, sources, dim, gamma, gx=0.0, gy=0.0, gz=0.0, cl=2, cq=1,
                 eta_crit=0.5, eta_fold=0.2, tol=0.5):
        self.dim = dim
        self.gamma = gamma
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.cl = cl
        self.cq = cq
        self.eta_crit = eta_crit
        self.eta_fold = eta_fold
        self.tol = tol
        super(EnergyEquation, self).__init__(dest, sources)


class StateEquation(Equation):
    """crksph.py:786-801: p = (gamma - 1) rho e"""

    def __init__(self, dest, sources, gamma):
        self.gamma = gamma
        super(StateEquation, self).__init__(dest, sources)


class SpeedOfSound(Equation):
    """crksph.py:804-810: cs = sqrt(gamma p / rho)"""

    def __init__(self, dest, sources=None, gamma=7.0):
        self.gamma = gamma
        super(SpeedOfSound, self).__init__(dest, sources)


class CRKSPHUpdateGhostProps(Equation):
    """crksph.py:813-844: copies to ghost particles, which the device has none of"""

    def __init__(self, dest, sources=None, dim=2):
        self.dim = dim
        super(CRKSPHUpdateGhostProps, self).__init__(dest, sources)


CRKSPH_PROPS = ('e', 'au', 'av', 'aw', 'ae', 'u0', 'v0', 'w0', 'cs', 'V', 'rhofac', 'x0', 'y0',
                'z0', 'rho0', 'ax', 'ay', 'az', 'arho')
CRKSPH_STRIDED = (('bi', 3), ('gradai', 3), ('gradbi', 9), ('gradv', 9))


def get_particle_array_crksph(constants=None, **props):
    """crksph.py:847-863"""
    pa = get_particle_array(additional_props=CRKSPH_PROPS, constants=constants, **props)
    pa.add_property('cwij')
    pa.add_property('ai')
    for name, stride in CRKSPH_STRIDED:
        pa.add_property(name, stride=stride)
    pa.set_output_arrays(pa.output_property_arrays + [p for p in ('p', 'V')
                                                      if p not in pa.output_property_arrays])
    return pa


class CRKSPHScheme(object):
    def __init__(self, fluids, dim, rho0, c0, nu, h0, p0, gx=0.0, gy=0.0, gz=0.0, cl=2, cq=1,
                 gamma=7.0, eta_crit=0.3, eta_fold=0.2, tol=0.5, has_ghosts=False):
        self.fluids = fluids
        self.solver = None
        self.dim = dim
        self.rho0 = rho0
        self.c0 = c0
        self.h0 = h0
        self.p0 = p0
        self.nu = nu
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.cl = cl
        self.cq = cq
        self.gamma = gamma
        self.eta_crit = eta_crit
        self.eta_fold = eta_fold
        self.tol = tol
        self.has_ghosts = has_ghosts

    def configure(self, **kw):                          # scheme.py: Scheme.configure
        for k, v in kw.items():
            if not hasattr(self, k):
                raise RuntimeError('Parameter {param} not defined for {scheme}.'
                                   .format(param=k, scheme=self.__class__.__name__))
            setattr(self, k, v)

    def get_steppers(self):                             # configure_solver, crksph.py:956-963
        return dict((f, CRKSPHStep()) for f in self.fluids)

    def get_equations(self):                            # crksph.py:978-1126
        all_ = self.fluids
        fl = self.fluids

        def ghosts(stage):
            if self.has_ghosts:
                stage.append(Group(equations=[CRKSPHUpdateGhostProps(dest=f, sources=None,
                                                                     dim=self.dim) for f in fl],
                                   real=False))

        def eos():
            eqs = []
            for f in fl:
                eqs.append(StateEquation(dest=f, sources=None, gamma=self.gamma))
                eqs.append(SpeedOfSound(dest=f, sources=None, gamma=self.gamma))
            return Group(equations=eqs)

        def sym(f):
            return CRKSPHSymmetric(dest=f, sources=all_, dim=self.dim, tol=self.tol)

        stage1 = [eos(),
                  Group(equations=[CRKSPHUpdateGhostProps(dest=f, sources=None, dim=self.dim)
                                   for f in fl], real=False),
                  Group(equations=[NumberDensity(dest=f, sources=all_) for f in fl], real=False)]
        ghosts(stage1)
        stage1.append(Group(equations=[CRKSPHPreStep(dest=f, sources=all_, dim=self.dim)
                                       for f in fl], real=False))
        ghosts(stage1)
        eq2 = []
        for f in fl:
            eq2.extend([sym(f), SummationDensityCRKSPH(dest=f, sources=all_)])
        stage1.append(Group(equations=eq2, real=False))
        stage1.append(eos())
        ghosts(stage1)
        eq4 = []
        for f in fl:
            eq4.extend([sym(f), VelocityGradient(dest=f, sources=all_, dim=self.dim)])
        stage1.append(Group(equations=eq4))
        ghosts(stage1)
        eq5 = []
        for f in fl:
            eq5.append(sym(f))
            eq5.append(MomentumEquation(dest=f, sources=all_, dim=self.dim, gx=self.gx,
                                        gy=self.gy, gz=self.gz, cl=self.cl, cq=self.cq,
                                        eta_crit=self.eta_crit, eta_fold=self.eta_fold))
            if abs(self.nu) > 1e-14:
                eq5.append(LaminarViscosity(dest=f, sources=self.fluids, nu=self.nu))
        stage1.append(Group(equations=eq5))

        stage2 = []
        ghosts(stage2)
        eq6 = []
        for f in fl:
            eq6.append(sym(f))
            eq6.append(EnergyEquation(dest=f, sources=all_, dim=self.dim, gamma=self.gamma))
        stage2.append(Group(equations=eq6))
        return MultiStageEquations([stage1, stage2])

    def setup_properties(self, particles, clean=True):  # crksph.py:1128-1153
        import numpy as np
        by_name = dict((p.name, p) for p in particles)
        for name in self.fluids:
            pa = by_name[name]
            for p in CRKSPH_PROPS + ('cwij', 'ai'):
                if p not in pa.properties:
                    pa.add_property(p)
            for p, stride in CRKSPH_STRIDED:
                if p not in pa.properties:
                    pa.add_property(p, stride=stride)
            if 'orig_idx' not in pa.properties:
                pa.add_property('orig_idx', type='int')
            pa.properties['orig_idx'][:] = np.arange(pa.get_number_of_particles())
            out = list(pa.output_property_arrays or
                       ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'm', 'h', 'pid', 'gid', 'tag'])
            pa.set_output_arrays(out + [p for p in ('p', 'V', 'e') if p not in out])


def make_crksph_solver(particles, scheme, kernel, dt, domain=None, device=0, **solver_kw):
    """A solver for a :class:`CRKSPHScheme` as its configure_solver makes it (crksph.py:936-976):
    CRKSPHIntegrator with CRKSPHStep for every fluid.  The arrays carry no dt_cfl / dt_force, so
    dt stays fixed."""
    from .solver import B200Solver
    integ = CRKSPHIntegrator(**scheme.get_steppers())
    kw = dict(adaptive_timestep=False, tf=1e9, fixed_h=True, device=device, domain=domain)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integ, dt=dt, **kw)
