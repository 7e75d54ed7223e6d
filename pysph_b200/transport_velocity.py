"""Equation descriptors of pysph/sph/wc/transport_velocity.py that the EDAC scheme's
internal-flow branch uses (class names and constructor arguments as there; the loop
bodies are ``k_tvf_pass1`` / ``k_tvf_pass2`` in csrc/b200sph.cu)."""
from .equations import Equation


class SummationDensity(Equation):
    """V = sum_b W_ab, rho = m_a V (transport_velocity.py:24-58).  Recognised by
    its MODULE: the class of the same name in basic_equations sums m_b W_ab."""


class MomentumEquationViscosity(Equation):
    """transport_velocity.py:328-386"""

    def __init__(self, dest, sources, nu):
        self.nu = nu
        super(MomentumEquationViscosity, self).__init__(dest, sources)


class MomentumEquationArtificialViscosity(Equation):
    """transport_velocity.py:389-448"""

    def __init__(self, dest, sources, c0, alpha=0.1):
        self.alpha = alpha
        self.c0 = c0
        super(MomentumEquationArtificialViscosity, self).__init__(dest, sources)


class MomentumEquationArtificialStress(Equation):
    """transport_velocity.py:451-545"""


class VolumeSummation(Equation):
    """V = sum_b W_ab (transport_velocity.py:61-75); the EDAC scheme applies it to its solid
    walls with every array as a source (wc/edac.py:817)."""


class SolidWallNoSlipBC(Equation):
    """transport_velocity.py:548-638: the viscous force on a fluid from a wall whose dummy
    velocity ug vg wg SetWallVelocity has extrapolated."""

    def __init__(self, dest, sources, nu):
        self.nu = nu
        super(SolidWallNoSlipBC, self).__init__(dest, sources)


class SetWallVelocity(Equation):
    """transport_velocity.py:84-134: uf = the fluid velocity extrapolated to the wall, ug = 2 u - uf
    (GTVFScheme's; the EDAC scheme has its own, wc/edac.py:186-230)"""


class ContinuitySolid(Equation):
    """transport_velocity.py:157-173: the continuity equation over a wall's dummy velocity ug"""


class StateEquation(Equation):
    """transport_velocity.py:176-216: p = p0 (rho / rho0 - b)"""

    def __init__(self, dest, sources, p0, rho0, b=1.0):
        self.b = b
        self.p0 = p0
        self.rho0 = rho0
        super(StateEquation, self).__init__(dest, sources)


class SolidWallPressureBC(Equation):
    """transport_velocity.py:641-736: the fluid pressure extrapolated to a wall particle, and the
    wall's density from it, rho = rho0 (p / p0 + b) (NOT wc/edac.py's: recognised by its module)"""

    def __init__(self, dest, sources, rho0, p0, b=1.0, gx=0.0, gy=0.0, gz=0.0):
        self.rho0 = rho0
        self.p0 = p0
        self.b = b
        self.gx = gx
        self.gy = gy
        self.gz = gz
        super(SolidWallPressureBC, self).__init__(dest, sources)
