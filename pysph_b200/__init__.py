"""pysph_b200 -- H100-native (sm_90a) evaluator for PySPH's WCSPH hot path.

The product is ``libb200sph.so`` (hand-written CUDA behind the C-ABI of
``include/b200sph.h``) plus the thin Python adapters in this package that
mirror the reference's plugin seam for this path:

==========================  ==================================================
reference (pypr/pysph)      here
==========================  ==================================================
compiled AccelerationEval   :class:`B200AccelerationEval`
compiled Integrator         :class:`PECIntegrator`, :class:`EPECIntegrator`,
                            :class:`TVDRK3Integrator`, :class:`EulerIntegrator`,
                            :class:`GTVFIntegrator`, :class:`CRKSPHIntegrator`
NNPS (LinkedListNNPS)       :class:`B200NNPS`
DeviceHelper (``pa.gpu``)   :class:`B200DeviceHelper` / :class:`B200Backend`
Equation / Group            :mod:`pysph_b200.equations`
WCSPHScheme.get_equations   :class:`pysph_b200.scheme.WCSPHScheme`
IISPHScheme.get_equations   :class:`pysph_b200.iisph.IISPHScheme`
GTVFScheme.get_equations    :class:`pysph_b200.gtvf.GTVFScheme` (a MultiStageEquations)
CRKSPHScheme.get_equations  :class:`pysph_b200.crksph.CRKSPHScheme` (a MultiStageEquations)
Solver step loop            :class:`B200Solver`
solver tools                :class:`DensityCorrection`, :class:`ShiftPositions`
tools.interpolator          :class:`Interpolator`
ParallelManager             :class:`pysph_b200.parallel.SlabParallelManager`
==========================  ==================================================

There is no CPU fallback: importing the adapters is cheap, but creating a
backend needs the built library and a CUDA device.
"""
from .particle_array import (ParticleArray, get_particle_array,
                             get_particle_array_wcsph, get_particle_array_edac,
                             get_particle_array_edac_wall, get_particle_array_edac_ext,
                             get_particle_array_elastic_dynamics)
from .kernels import CubicSpline, WendlandQuintic, QuinticSpline, Gaussian
from .equations import (Equation, Group, SummationDensity, ContinuityEquation, LaminarViscosity,
                        MonaghanArtificialViscosity, XSPHCorrection, TaitEOS,
                        TaitEOSHGCorrection, MomentumEquation,
                        UpdateSmoothingLengthFerrari, ShepardFilter, MLSFirstOrder2D,
                        MLSFirstOrder3D)
from .scheme import WCSPHScheme
from .backend import B200Backend, B200DeviceHelper
from .domain import DomainManager
from .nnps import B200NNPS
from .acceleration_eval import B200AccelerationEval
from .integrator import (B200Integrator, PECIntegrator, EPECIntegrator,
                         TVDRK3Integrator, EulerIntegrator, WCSPHStep, WCSPHTVDRK3Step)
from .solver import B200Solver
from .tools import Tool, DensityCorrection
from .shift import SimpleShift, FickianShift, CorrectVelocities, ShiftPositions
from .interpolator import Interpolator, get_bounding_box, get_nx_ny_nz
from .edac import EDACScheme, EDACTVFStep, EDACStep
from .output import dump, load
from .solid_mech import ElasticSolidsScheme, SolidMechStep
from .iisph import (IISPHScheme, IISPHStep, get_particle_array_iisph, make_iisph_solver,
                    last_iterations)
from .equations import MultiStageEquations
from .gtvf import (GTVFScheme, GTVFStep, GTVFIntegrator, get_particle_array_gtvf,
                   make_gtvf_solver)
from .crksph import (CRKSPHScheme, CRKSPHStep, CRKSPHIntegrator, get_particle_array_crksph,
                     make_crksph_solver)

__version__ = '0.1.0'


def make_wcsph_solver(particles, params, kernel, device=0, **solver_kw):
    """Build a ready-to-step WCSPH solver from the parameter dict returned by
    ``geometry.dam_break_3d_params`` / ``dam_break_2d_params``."""
    p = dict(params)
    integ_name = p.pop('integrator', 'EPEC')
    dt0 = p.pop('dt0')
    n_damp = p.pop('n_damp', 0)
    cfl = p.pop('cfl', 0.3)
    scheme = WCSPHScheme(**p)
    names = scheme.fluids + scheme.solids
    cls = {'EPEC': EPECIntegrator, 'PEC': PECIntegrator,
           'TVDRK3': TVDRK3Integrator}[integ_name]
    # WCSPHScheme.configure_solver (scheme.py:360-386): TVD-RK3 steps every array with
    # WCSPHTVDRK3Step
    step_cls = WCSPHTVDRK3Step if cls is TVDRK3Integrator else WCSPHStep
    integrator = cls(**dict((n, step_cls()) for n in names))
    kw = dict(adaptive_timestep=True, cfl=cfl, n_damp=n_damp, tf=1e9,
              fixed_h=not p.get('update_h', False), device=device)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integrator,
                      dt=dt0, **kw)


def make_edac_solver(particles, scheme, kernel, dt, domain=None, integrator='PEC',
                     device=0, **solver_kw):
    """Fixed-dt solver for an :class:`EDACScheme` (the reference's configure_solver
    default is PECIntegrator + EDACTVFStep, wc/edac.py:657-702)."""
    cls = {'EPEC': EPECIntegrator, 'PEC': PECIntegrator}[integrator]
    integ = cls(**scheme.get_steppers())
    kw = dict(adaptive_timestep=False, tf=1e9, fixed_h=True, device=device,
              domain=domain)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integ, dt=dt, **kw)


def make_elastic_solver(particles, scheme, kernel, dt, integrator='EPEC', device=0,
                        **solver_kw):
    """Fixed-dt solver for an :class:`ElasticSolidsScheme` (configure_solver's default
    is EPECIntegrator + SolidMechStep, solid_mech/basic.py:653-684)."""
    cls = {'EPEC': EPECIntegrator, 'PEC': PECIntegrator}[integrator]
    integ = cls(**scheme.get_steppers())
    kw = dict(adaptive_timestep=False, tf=1e9, fixed_h=True, device=device)
    kw.update(solver_kw)
    return B200Solver(particles, scheme.get_equations(), kernel, integ, dt=dt, **kw)
