"""The cost of IISPHScheme on the flagship geometry: the 3-D dam break of `bench.py` (SPHERIC
test 2, dx = 0.00877: ~1.0 M fluid + ~0.23 M wall and obstacle particles, CubicSpline), one GPU.

    python bench_iisph.py [--dx 0.00877] [--steps 50] [--warmup 10] [--profile-steps 5]

Two arms in one process on one card:
  * IISPH: EulerIntegrator + IISPHStep with the adaptive dt of dam_break_2d.py's IISPH run
    (initial dt = 0.125 * 10 * h / c0, cfl 0.3), gravity, rho0 = 1000;
  * WCSPH: the flagship (EPEC + WCSPHStep, dam_break_3d.py's parameters, adaptive dt).
Each arm builds a fresh solver, runs `warmup` steps and times `steps` steps with CUDA events;
reported: ms per step, simulated seconds per wall-clock second, and the neighbour-search
counters of the timed window per step (full builds, light updates, list builds, deferred checks
that failed, proactive builds -- what the list skin controller did).  For IISPH also the
pressure iterations of every step of a second window (each read back, so not timed) and, from
torch.profiler in a run of its own, the mean device time per step of each pass.  The card name,
power limit and SM clock limit are read in the same process.  Prints one JSON line.  Needs a
CUDA device; writes nothing.
"""
import argparse
import json
import sys
import time

from bench_integrators import card

# k_iisph<K, DIM, PASS>: the pass names (csrc/iisph_kernels.cuh)
PASSES = ('V', 'rho', 'advection+dii', 'rho_adv+aii', 'dijpj', 'pressure_solve', 'pressure_force')


def make(dx, arm):
    import numpy as np
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    params = geo.dam_break_3d_params(dx)
    if arm == 'wcsph':
        return pb.make_wcsph_solver(pas, params, pb.CubicSpline(dim=3)), pas
    arrays = [pb.get_particle_array_iisph(
        name=pa.name, **dict((k, pa.properties[k].copy()) for k in ('x', 'y', 'z', 'h', 'm', 'rho', 'gid')))
        for pa in pas]
    sch = pb.IISPHScheme(['fluid'], ['boundary', 'obstacle'], 3, params['rho0'], gz=-9.81)
    h = params['h0']
    c0 = 10.0 * np.sqrt(2.0 * 9.81 * 0.55)
    s = pb.make_iisph_solver(arrays, sch, pb.CubicSpline(dim=3), 0.125 * 10 * h / c0,
                             adaptive_timestep=True, cfl=0.3)
    return s, arrays


def timed_run(dx, arm, steps, warmup):
    import torch
    s, pas = make(dx, arm)
    be = s.backend
    stream = torch.cuda.current_stream()
    be.use_torch_stream(stream)
    s.initialise()
    for _ in range(warmup):
        s.step()
    t0, dt0 = s.t, s.dt
    be.ctx.call('b200sph_reset_stats')
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        s.step()
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    st = be.stats()
    t1 = s.t
    out = dict(particles=int(sum(pa.get_number_of_particles() for pa in pas)),
               ms_per_step=ms / steps, simulated_s=t1 - t0,
               sim_s_per_wall_s=(t1 - t0) / (ms * 1e-3), dt_first=dt0, dt_last=s.dt)
    for k in ('full_builds', 'light_updates', 'list_builds', 'deferred_failed', 'proactive_builds'):
        out[k + '_per_step'] = st[k] / float(steps)
    if arm == 'iisph':
        import pysph_b200 as pb
        its = []
        for _ in range(steps):
            s.step()
            its.append(pb.last_iterations(s)[0])
        out['iterations'] = dict(mean=sum(its) / float(len(its)), min=min(its), max=max(its),
                                 per_step=its)
    return out


def pass_ms(dx, steps, warmup):
    """mean device time per step of each IISPH pass and of the rest, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    s, _ = make(dx, 'iisph')
    s.backend.use_torch_stream(torch.cuda.current_stream())
    s.initialise()
    for _ in range(warmup):
        s.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            s.step()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.replace('void ', '')
        if name.startswith('k_iisph<'):
            key = PASSES[int(name.split('<')[1].split('>')[0].split(',')[2])]
        else:
            key = name.split('(')[0].split('<')[0]
        per[key] = per.get(key, 0.0) + e.device_time / 1e3
    return dict((k, v / steps) for k, v in sorted(per.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--dx', type=float, default=0.00877)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_iisph.py: no CUDA device (there is no CPU fallback)')
    info = card()
    res = dict((arm, timed_run(args.dx, arm, args.steps, args.warmup)) for arm in ('iisph', 'wcsph'))
    res['iisph']['device_ms_per_step'] = pass_ms(args.dx, args.profile_steps, args.warmup)
    print(json.dumps(dict(workload='dam_break_3d dx=%g CubicSpline' % args.dx, steps=args.steps,
                          warmup=args.warmup, gpu=info, arms=res, date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
