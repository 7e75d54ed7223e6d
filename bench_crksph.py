"""The cost of CRKSPHScheme against EDAC on the 3-D Taylor-Green vortex, one GPU.

    python bench_crksph.py [--tg-nx 126] [--steps 30] [--warmup 5] [--rounds 2]
                           [--profile-steps 3]

The periodic 3-D Taylor-Green vortex of taylor_green.py, nx^3 particles (2.0 M at nx = 126),
QuinticSpline, Re = 100, the example's fixed dt: CRKSPH (CRKSPHIntegrator) against EDAC
(PECIntegrator + EDACTVFStep, the example's default scheme).  The CRKSPH fluid starts with
e = c0^2 / (gamma (gamma - 1)), so that its sound speed is the EDAC arm's c0: with e = 0, as
taylor_green.py runs it, e drifts below zero within steps at this resolution and
cs = sqrt(gamma p / rho) turns NaN, as the reference's SpeedOfSound does.
Both solvers are built once; each round times `steps` steps of one and then of the other with CUDA
events (ms per step), after `warmup` steps each, so that the two arms alternate in one process.
The CRKSPH arm also gets the mean device time per step of each pass from torch.profiler, in a
window of its own.  The card name, power limit and SM clock limit are read in the same process.
Prints one JSON line.  Needs a CUDA device; writes nothing.
"""
import argparse
import json
import sys
import time

from bench_integrators import card

# k_crksph<K, DIM, PASS>: the pass names (csrc/crksph_kernels.cuh)
PASSES = ('number_density', 'pre_step', 'density', 'velocity_gradient', 'momentum', 'energy')


def make(arm, nx):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    p = geo.taylor_green_params(nx, dim=3)
    e = geo.taylor_green_particles(nx, dim=3, perturb=0.1)
    dom = pb.DomainManager(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, zmin=0.0, zmax=1.0,
                           periodic_in_x=True, periodic_in_y=True, periodic_in_z=True)
    k = pb.QuinticSpline(dim=3)
    if arm == 'edac':
        sch = pb.EDACScheme(['fluid'], [], 3, p['c0'], p['nu'], p['rho0'], pb=p['pb'], h=p['h'])
        return pb.make_edac_solver([e], sch, k, p['dt'], domain=dom), [e]
    pa = pb.get_particle_array_crksph(name='fluid', **dict(
        (n, e.properties[n].copy()) for n in ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'gid')))
    sch = pb.CRKSPHScheme(['fluid'], 3, p['rho0'], p['c0'], p['nu'], p['h'], 0.0)
    sch.setup_properties([pa])
    pa.e[:] = p['c0'] ** 2 / (sch.gamma * (sch.gamma - 1.0))
    return pb.make_crksph_solver([pa], sch, k, p['dt'], domain=dom), [pa]


def window(s, steps):
    import torch
    stream = torch.cuda.current_stream()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        s.step()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def pass_ms(s, steps):
    """mean device time per step of each CRKSPH pass and of the rest, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
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
        if name.startswith('k_crksph<'):
            key = PASSES[int(name.split('<')[1].split('>')[0].split(',')[2])]
        else:
            key = name.split('(')[0].split('<')[0]
        per[key] = per.get(key, 0.0) + e.device_time / 1e3
    return dict((k, v / steps) for k, v in sorted(per.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--tg-nx', type=int, default=126)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--profile-steps', type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_crksph.py: no CUDA device (there is no CPU fallback)')
    info = card()
    solvers, times = {}, {}
    for arm in ('crksph', 'edac'):
        s, pas = make(arm, args.tg_nx)
        s.backend.use_torch_stream(torch.cuda.current_stream())
        s.initialise()
        for _ in range(args.warmup):
            s.step()
        solvers[arm] = (s, int(sum(pa.get_number_of_particles() for pa in pas)))
        times[arm] = []
    for _ in range(args.rounds):
        for arm in ('crksph', 'edac'):
            times[arm].append(window(solvers[arm][0], args.steps))
    res = dict((arm, dict(particles=solvers[arm][1], ms_per_step=min(times[arm]),
                          ms_per_step_rounds=times[arm], dt=solvers[arm][0].dt))
               for arm in ('crksph', 'edac'))
    res['crksph']['device_ms_per_step'] = pass_ms(solvers['crksph'][0], args.profile_steps)
    res['crksph_over_edac'] = res['crksph']['ms_per_step'] / res['edac']['ms_per_step']
    print(json.dumps(dict(steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          tg_nx=args.tg_nx, gpu=info, tg3d=res, date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
