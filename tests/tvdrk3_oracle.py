"""TEST INFRASTRUCTURE: TVD-RK3 on the fp64 oracle.

TVDRK3Integrator.one_timestep (pysph/sph/integrator.py:441-460) around the oracle's WCSPH
evaluation (oracle.WCSPHOracleSolver: the loops, the NNPS and the time step), with the
stages of WCSPHTVDRK3Step (pysph/sph/integrator_step.py:96-168) restated in numpy fp64 on
the real particles of the oracle's arrays, in place -- the oracle library reads and writes
those same buffers.
"""
from oracle import oracle as orc

# (q, q0, aq) of WCSPHTVDRK3Step
STATE = (('u', 'u0', 'au'), ('v', 'v0', 'av'), ('w', 'w0', 'aw'),
         ('x', 'x0', 'ax'), ('y', 'y0', 'ay'), ('z', 'z0', 'az'),
         ('rho', 'rho0', 'arho'))


def stage_rk3(pa, which, dt):
    """initialize (0) / stage1 / stage2 / stage3 of WCSPHTVDRK3Step over the real particles
    of one array, in the reference's association order"""
    n = pa.num_real_particles
    props = pa.properties
    for q, q0, aq in STATE:
        a, a0, acc = props[q][:n], props[q0][:n], props[aq][:n]
        if which == 0:
            a0[:] = a
        elif which == 1:
            a[:] = a0 + dt * acc
        elif which == 2:
            a[:] = 0.75 * a0 + 0.25 * (a + dt * acc)
        else:
            a[:] = (1. / 3.) * a0 + (2. / 3.) * (a + dt * acc)


class TVDRK3OracleSolver(orc.WCSPHOracleSolver):
    """WCSPHOracleSolver stepping with TVDRK3Integrator + WCSPHTVDRK3Step (no periodic
    domain: the device refuses one under TVD-RK3)."""

    def __init__(self, particles, params, kernel='CubicSpline', threads=1):
        orc.WCSPHOracleSolver.__init__(self, particles, dict(params, integrator='TVDRK3'),
                                       kernel, threads=threads)

    def _stage(self, which, dt):
        for a in self.all:
            stage_rk3(self.o.pas[a], which, dt)

    def one_timestep(self, dt):
        self._stage(0, 0.0)
        for which in (1, 2, 3):
            self.compute_accelerations()
            self._stage(which, dt)
            self.update_domain()
