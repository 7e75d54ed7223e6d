"""The cost of GTVFScheme against the schemes users pick beside it, one GPU.

    python bench_gtvf.py [--tg-nx 126] [--dam-dx 0.0014] [--steps 50] [--warmup 10]
                         [--profile-steps 5]

Two workloads, each timed against its baseline in the same process on the same card:
  * tg3d: the periodic 3-D Taylor-Green vortex of taylor_green.py, nx^3 particles (2.0 M at
    nx = 126), QuinticSpline, Re = 100, the example's fixed dt: GTVF (GTVFIntegrator) against
    EDAC (PECIntegrator + EDACTVFStep, the example's default scheme);
  * dam2d: dam_break_2d.py's tank (4 wall layers) and 1 x 2 column at dx (~1.1 M particles at
    dx = 0.0014), QuinticSpline, dt = 0.125 h / c0: GTVF against WCSPH (PEC + WCSPHStep, the
    example's default scheme, adaptive dt).
Each arm builds a fresh solver, runs `warmup` steps and times `steps` steps with CUDA events
(ms per step).  The GTVF arms also get the mean device time per step of each pass from
torch.profiler, in a run of its own.  The card name, power limit and SM clock limit are read in
the same process.  Prints one JSON line.  Needs a CUDA device; writes nothing.
"""
import argparse
import json
import sys
import time

from bench_integrators import card

# k_gtvf<K, DIM, PASS>: the pass names (csrc/gtvf_kernels.cuh)
PASSES = ('wall_velocity', 'continuity', 'correct_density', 'wall_pressure', 'momentum')


def make(workload, arm, size):
    import numpy as np
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    if workload == 'tg3d':
        p = geo.taylor_green_params(size, dim=3)
        e = geo.taylor_green_particles(size, dim=3, perturb=0.1)
        dom = pb.DomainManager(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, zmin=0.0, zmax=1.0,
                               periodic_in_x=True, periodic_in_y=True, periodic_in_z=True)
        k = pb.QuinticSpline(dim=3)
        if arm == 'edac':
            sch = pb.EDACScheme(['fluid'], [], 3, p['c0'], p['nu'], p['rho0'], pb=p['pb'], h=p['h'])
            return pb.make_edac_solver([e], sch, k, p['dt'], domain=dom), [e]
        pa = pb.get_particle_array_gtvf(name='fluid', **dict(
            (n, e.properties[n].copy()) for n in ('x', 'y', 'z', 'u', 'v', 'w', 'h', 'm', 'rho', 'gid')))
        sch = pb.GTVFScheme(['fluid'], [], 3, p['rho0'], p['c0'], p['nu'], p['h'], p['c0'] ** 2 * p['rho0'])
        return pb.make_gtvf_solver([pa], sch, k, p['dt'], domain=dom), [pa]
    dx = size
    k = pb.QuinticSpline(dim=2)
    if arm == 'wcsph':
        pas = geo.dam_break_2d_particles(dx)
        for pa in pas:                     # h = hdx dx, m = rho0 dx^2 at this resolution
            pa.h[:] = 1.3 * dx
            pa.m[:] = dx * dx * 1000.0
        params = dict(geo.dam_break_2d_params(dx), h0=1.3 * dx)
        return pb.make_wcsph_solver(pas, params, k), pas
    from pysph_b200.geometry import _block_2d, _tank_2d
    h, rho0 = 1.3 * dx, 1000.0
    c0 = 10.0 * np.sqrt(2 * 9.81 * 2.0)
    xt, yt = _tank_2d(dx, 4.0, 4.0, 4, [2, 0])
    xf, yf = _block_2d(dx, 1.0, 2.0, [0.5, 1])
    fluid = pb.get_particle_array_gtvf(name='fluid', x=xf + dx, y=yf + dx, h=h, m=dx * dx * rho0,
                                       rho=rho0)
    wall = pb.get_particle_array(name='boundary', x=xt, y=yt, h=h, m=dx * dx * rho0, rho=rho0)
    sch = pb.GTVFScheme(['fluid'], ['boundary'], 2, rho0, c0, 0.0, h, c0 * c0 * rho0, gy=-9.81)
    sch.setup_properties([fluid, wall])
    return pb.make_gtvf_solver([fluid, wall], sch, k, 0.125 * h / c0), [fluid, wall]


def timed_run(workload, arm, size, steps, warmup):
    import torch
    s, pas = make(workload, arm, size)
    stream = torch.cuda.current_stream()
    s.backend.use_torch_stream(stream)
    s.initialise()
    for _ in range(warmup):
        s.step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        s.step()
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    return dict(particles=int(sum(pa.get_number_of_particles() for pa in pas)),
                ms_per_step=ms / steps, dt=s.dt)


def pass_ms(workload, size, steps, warmup):
    """mean device time per step of each GTVF pass and of the rest, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    s, _ = make(workload, 'gtvf', size)
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
        if name.startswith('k_gtvf<'):
            key = PASSES[int(name.split('<')[1].split('>')[0].split(',')[2])]
        else:
            key = name.split('(')[0].split('<')[0]
        per[key] = per.get(key, 0.0) + e.device_time / 1e3
    return dict((k, v / steps) for k, v in sorted(per.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--tg-nx', type=int, default=126)
    ap.add_argument('--dam-dx', type=float, default=0.0014)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_gtvf.py: no CUDA device (there is no CPU fallback)')
    info = card()
    res = {}
    for workload, size, base in (('tg3d', args.tg_nx, 'edac'), ('dam2d', args.dam_dx, 'wcsph')):
        arms = dict((arm, timed_run(workload, arm, size, args.steps, args.warmup))
                    for arm in ('gtvf', base))
        arms['gtvf']['device_ms_per_step'] = pass_ms(workload, size, args.profile_steps, args.warmup)
        arms['gtvf_over_' + base] = arms['gtvf']['ms_per_step'] / arms[base]['ms_per_step']
        res[workload] = arms
    print(json.dumps(dict(steps=args.steps, warmup=args.warmup, tg_nx=args.tg_nx,
                          dam_dx=args.dam_dx, gpu=info, workloads=res,
                          date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
