"""tests/test_gpu_tvdrk3.py on the library emulation (the loader of test_library_on_cpu.py),
smaller, where no GPU is available; the integrator's refusals, which need no library; and
the slab decomposition under TVD-RK3 on three ranks over gloo."""
import os

import numpy as np
import pytest

import test_gpu_tvdrk3 as t
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

DX = 0.08


def test_stepper_golden_emulated(emulated_library):
    t.check_stepper_golden()


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_fused_is_bitwise_unfused_emulated(emulated_library, monkeypatch, records, device_dt):
    t.check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx=DX, steps=20)


@pytest.mark.parametrize('vscale', [0.0, 3.0])
def test_dam_break_3d_vs_oracle_emulated(emulated_library, vscale):
    st = t.check_dam_break_3d_vs_oracle(dx=DX, steps=20, vscale=vscale)
    if vscale:
        assert st['full_builds'] >= 2, st


def test_dam_break_2d_gate_vs_oracle_emulated(emulated_library):
    t.check_dam_break_2d_gate_vs_oracle(dx=0.06, steps=20)


@pytest.mark.parametrize('device_dt', [True, False])
def test_dt_from_the_third_evaluation_emulated(emulated_library, device_dt):
    t.check_dt_comes_from_the_third_evaluation(dx=DX, device_dt=device_dt)


def test_device_dt_is_bitwise_host_dt_emulated(emulated_library):
    t.check_device_dt_is_bitwise_host_dt(dx=DX, steps=12)


def test_post_stage_times_emulated(emulated_library):
    t.check_post_stage_times(dx=DX)


def test_forced_repeats_change_nothing_emulated(emulated_library):
    t.check_forced_repeats_change_nothing(dx=DX, steps=4)


def test_restart_vs_oracle_emulated(emulated_library, tmp_path):
    t.check_restart_vs_oracle(tmp_path, dx=DX, steps_before=6, steps_after=5)


def test_refusals_on_the_library_emulated(emulated_library):
    t.check_refusals_on_the_library()


def test_integrators_accept_only_their_steppers():
    """TVDRK3Integrator takes WCSPHTVDRK3Step only; PEC / EPEC refuse it; a periodic domain is
    refused under TVD-RK3 when the NNPS is attached."""
    import pysph_b200 as pb
    pb.TVDRK3Integrator(fluid=pb.WCSPHTVDRK3Step(), wall=pb.WCSPHTVDRK3Step())
    for stepper in (pb.WCSPHStep(), pb.EDACTVFStep(), pb.SolidMechStep()):
        with pytest.raises(NotImplementedError, match='TVDRK3Integrator'):
            pb.TVDRK3Integrator(fluid=stepper)
    for cls in (pb.PECIntegrator, pb.EPECIntegrator):
        with pytest.raises(NotImplementedError, match='WCSPHTVDRK3Step'):
            cls(fluid=pb.WCSPHTVDRK3Step())
        cls(fluid=pb.WCSPHStep())
    integ = pb.TVDRK3Integrator(fluid=pb.WCSPHTVDRK3Step())

    class NNPS(object):
        domain = pb.DomainManager(xmin=0.0, xmax=1.0, periodic_in_y=True, ymax=1.0)
    with pytest.raises(NotImplementedError, match='periodic'):
        integ.set_nnps(NNPS())
    NNPS.domain = pb.DomainManager(xmin=0.0, xmax=1.0, mirror_in_x=True)
    integ.set_nnps(NNPS())


# ---- the slab decomposition on three ranks -----------------------------------------------------
SLAB_DX, SLAB_STEPS = 0.07, 8


def _slab_worker(rank, world, port, so, q):
    import torch
    import torch.distributed as dist
    from pysph_b200 import _lib
    _lib.LIB_PATH, _lib._lib = so, None
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo, parallel
    import test_gpu_multi as M

    Base = parallel.DeviceHaloOps

    class HostHaloOps(Base):
        """DeviceHaloOps with CPU tensors: under the emulation device memory IS host memory"""

        def __init__(self, backend, device):
            Base.__init__(self, backend, 0)
            self.device = torch.device('cpu')

        def read_later(self, tensor):
            v = float(tensor[0])
            return lambda: v
    parallel.DeviceHaloOps = HostHaloOps
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    os.environ['B200SPH_PEER_HALO'] = '0'
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        params = dict(geo.dam_break_3d_params(SLAB_DX), integrator='TVDRK3')
        solver, pm, pas = parallel.make_slab_solver(SLAB_DX, params, pb.CubicSpline(dim=3),
                                                    rank, world, device=0, n_damp=0)
        assert isinstance(solver.integrator, pb.TVDRK3Integrator)
        M._perturb(pas)
        solver.backend.push_all()
        for _ in range(SLAB_STEPS):
            solver.step()
        t_end = solver.t
        solver.pull()
        q.put((rank, M._collect(pas), pm.n_full, pm.n_refresh, t_end))
    except Exception:
        import traceback
        q.put(('error', rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def test_slabs_match_one_process_emulated(emulated_library):
    """Three x-slabs (one rank with two neighbours), adaptive device-resident dt, particles
    migrating across the cuts between stages: equal to the one-process run by gid."""
    import socket
    import torch.multiprocessing as mp
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo, _lib
    import test_gpu_multi as M
    world = 3
    params = dict(geo.dam_break_3d_params(SLAB_DX), integrator='TVDRK3', n_damp=0)
    pas = geo.dam_break_3d_particles(dx=SLAB_DX)
    M._perturb(pas)
    s = t._solver(pas, params)
    assert isinstance(s.integrator, pb.TVDRK3Integrator)
    for _ in range(SLAB_STEPS):
        s.step()
    t_ref = s.t
    s.pull()
    ref = M._collect(pas)
    sock = socket.socket()
    sock.bind(('127.0.0.1', 0))
    port = sock.getsockname()[1]
    sock.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_slab_worker, args=(r, world, port, _lib.LIB_PATH, q))
             for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=900) for _ in range(world)]
    assert not any(o[0] == 'error' for o in out), [o[2] for o in out if o[0] == 'error'][:1]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    t.compare_slabs(out, ref, t_ref, params)
