"""Equation / Group descriptors for the WCSPH hot path.

These mirror the *interface* of the reference's plugin API for this path --
class names, constructor arguments and the plain attributes the code generator
reads from ``equation.__dict__`` (pysph/sph/equation.py:389-420, :885-892) --
but carry no loop bodies: on the B200 backend the bodies are the hand-written
CUDA of csrc/b200sph.cu.  ``pysph_b200.program`` recognises equations by class
name, so the reference's own objects (pysph.sph.wc.basic.MomentumEquation ...)
are accepted unchanged; an equation class the backend has no kernel for raises
NotImplementedError at setup, before the run starts (mirrors the reference's
pre-flight checks, pysph/sph/acceleration_eval.py:204-205).
"""
import itertools

_group_counter = itertools.count()


class Equation(object):
    """pysph/sph/equation.py:389-420"""

    def __init__(self, dest, sources):
        self.dest = dest
        if sources is not None and len(sources) > 0:
            self.sources = list(sources)
        else:
            self.sources = None
        self.no_source = self.sources is None
        self.name = self.__class__.__name__

    def __repr__(self):
        keys = [k for k in self.__dict__ if k not in ('name', 'no_source')]
        return '%s(%s)' % (self.name, ', '.join(
            '%s=%r' % (k, self.__dict__[k]) for k in keys))


class Group(object):
    """pysph/sph/equation.py:452-560 (attributes only)."""

    def __init__(self, equations, real=True, update_nnps=False, iterate=False,
                 max_iterations=1, min_iterations=0, pre=None, post=None,
                 condition=None, start_idx=0, stop_idx=None, name=None):
        self.real = real
        self.update_nnps = update_nnps
        self.iterate = iterate
        self.max_iterations = max_iterations
        self.min_iterations = min_iterations
        self.pre = pre
        self.post = post
        self.condition = condition
        self.start_idx = start_idx
        self.stop_idx = stop_idx
        self.name = name or 'Group_%d' % next(_group_counter)
        subs = [e for e in equations if isinstance(e, Group)]
        if subs and len(subs) != len(equations):
            raise ValueError(
                'All elements must be Groups if you use sub groups.')
        self.has_subgroups = len(subs) > 0
        self.equations = list(equations)


class MultiStageEquations(object):
    """pysph/sph/equation.py:966-995: one list of Groups per evaluation of a multi-stage
    integrator (GTVFIntegrator evaluates twice per step).  B200Solver builds one
    B200AccelerationEval per list, as make_acceleration_evals does (acceleration_eval.py:76-90)."""

    def __init__(self, groups):
        assert type(groups) in (list, tuple)
        self.groups = groups


class SummationDensity(Equation):
    """rho_a = sum_b m_b W_ab   (pysph/sph/basic_equations.py:19-29)"""


class ContinuityEquation(Equation):
    """arho_a = sum_b m_b v_ab . grad W_ab (pysph/sph/basic_equations.py:180-192)"""


class MonaghanArtificialViscosity(Equation):
    """pysph/sph/basic_equations.py:195-257"""

    def __init__(self, dest, sources, alpha=1.0, beta=1.0):
        self.alpha = alpha
        self.beta = beta
        super(MonaghanArtificialViscosity, self).__init__(dest, sources)


class XSPHCorrection(Equation):
    """pysph/sph/basic_equations.py:260-300"""

    def __init__(self, dest, sources, eps=0.5):
        self.eps = eps
        super(XSPHCorrection, self).__init__(dest, sources)


class LaminarViscosity(Equation):
    """pysph/sph/wc/viscosity.py:5-27 (WCSPHScheme(nu != 0), scheme.py:486-496)"""

    def __init__(self, dest, sources, nu, eta=0.01):
        self.nu = nu
        self.eta = eta
        super(LaminarViscosity, self).__init__(dest, sources)


class TaitEOS(Equation):
    """pysph/sph/wc/basic.py:9-65"""

    def __init__(self, dest, sources, rho0, c0, gamma, p0=0.0):
        self.rho0 = rho0
        self.rho01 = 1.0 / rho0
        self.c0 = c0
        self.gamma = gamma
        self.gamma1 = 0.5 * (gamma - 1.0)
        self.B = rho0 * c0 * c0 / gamma
        self.p0 = p0
        super(TaitEOS, self).__init__(dest, sources)


class TaitEOSHGCorrection(Equation):
    """pysph/sph/wc/basic.py:68-126"""

    def __init__(self, dest, sources, rho0, c0, gamma):
        self.rho0 = rho0
        self.rho01 = 1.0 / rho0
        self.c0 = c0
        self.gamma = gamma
        self.gamma1 = 0.5 * (gamma - 1.0)
        self.B = rho0 * c0 * c0 / gamma
        super(TaitEOSHGCorrection, self).__init__(dest, sources)


class MomentumEquation(Equation):
    """pysph/sph/wc/basic.py:129-269"""

    def __init__(self, dest, sources, c0, alpha=1.0, beta=1.0, gx=0.0, gy=0.0,
                 gz=0.0, tensile_correction=False):
        self.alpha = alpha
        self.beta = beta
        self.gx = gx
        self.gy = gy
        self.gz = gz
        self.c0 = c0
        self.tensile_correction = tensile_correction
        super(MomentumEquation, self).__init__(dest, sources)


class UpdateSmoothingLengthFerrari(Equation):
    """pysph/sph/wc/basic.py:417-463"""

    def __init__(self, dest, sources, dim, hdx):
        self.dim1 = 1. / dim
        self.hdx = hdx
        super(UpdateSmoothingLengthFerrari, self).__init__(dest, sources)


class ShepardFilter(Equation):
    """Zeroth-order density re-initialisation, wc/density_correction.py:7-46:
    rho_a = sum_b m_b W_ab / sum_b (m_b / rhotmp_b) W_ab"""


class MLSFirstOrder2D(Equation):
    """First-order moving-least-squares density re-initialisation in 2-D,
    wc/density_correction.py:49-140"""


class MLSFirstOrder3D(Equation):
    """First-order moving-least-squares density re-initialisation in 3-D,
    wc/density_correction.py:143-205"""
