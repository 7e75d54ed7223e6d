"""The cost of ShiftPositions on the benchmark's second workload: the periodic 3-D Taylor-Green
vortex as `bench.py --workload taylor_green` builds it (EDAC transport-velocity branch,
QuinticSpline, nx^3 particles in the periodic unit cube, PEC + EDACTVFStep at the example's fixed
dt), one GPU.

    python bench_shift.py [--nx 126] [--runs 3] [--steps 100] [--warmup 20] [--freq 10]

Four arms alternate, `runs` times each, in one process on one card: no tool, simple, fickian
and fickian + correct_velocity, every `freq` steps.  Every run builds a fresh solver, warms up
and times `steps` steps with CUDA events.  Reported per run: ms per step, shift calls and list
builds in the timed window; then, in a separate run of each shifting arm with torch.profiler,
the mean device time of the tool's kernels per call.  The card name, power limit and SM clock
limit are read in the same process.  Prints one JSON line.  Needs a CUDA device; writes nothing.
"""
import argparse
import json
import sys
import time

from bench_integrators import card

ARMS = (None, ('simple', False), ('fickian', False), ('fickian', True))
KERNELS = ('k_shift_pack', 'k_shift_vmax', 'k_shift', 'k_shift_apply', 'k_correct_velocities')


def arm_name(a):
    return 'none' if a is None else a[0] + ('+correct' if a[1] else '')


def make(nx, arm, freq):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    p = geo.taylor_green_params(nx, dim=3)
    pa = geo.taylor_green_particles(nx, dim=3)
    dm = pb.DomainManager(xmin=0, xmax=1, ymin=0, ymax=1, zmin=0, zmax=1,
                          periodic_in_x=True, periodic_in_y=True, periodic_in_z=True)
    sch = pb.EDACScheme(['fluid'], [], dim=3, c0=p['c0'], nu=p['nu'], rho0=p['rho0'],
                        pb=p['pb'], h=p['h'])
    s = pb.make_edac_solver([pa], sch, pb.QuinticSpline(dim=3), dt=p['dt'], domain=dm)
    tool = None
    if arm is not None:
        tool = pb.ShiftPositions(s, 'fluid', freq=freq, shift_kind=arm[0], correct_velocity=arm[1])
        s.add_tool(tool)
    return s, pa, tool


def timed_run(nx, arm, freq, steps, warmup):
    import torch
    s, pa, tool = make(nx, arm, freq)
    be = s.backend
    stream = torch.cuda.current_stream()
    be.use_torch_stream(stream)
    s.initialise()
    for _ in range(warmup):
        s.step()
    be.ctx.call('b200sph_reset_stats')
    count0 = tool.count if tool else 0
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        s.step()
    e1.record(stream)
    torch.cuda.synchronize()
    st = be.stats()
    calls = 0 if tool is None else sum(1 for c in range(count0, tool.count) if c % freq == 0)
    return dict(particles=int(pa.get_number_of_particles()), ms_per_step=e0.elapsed_time(e1) / steps,
                shift_calls=calls, list_builds=int(st['list_builds']), full_builds=int(st['full_builds']))


def tool_kernel_us(nx, arm, freq, steps, warmup):
    """device time of the tool's kernels per call, from torch.profiler (a run of its own)"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    s, _, _ = make(nx, arm, freq)
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
        name = e.name.split('(')[0].split('<')[0].replace('void ', '')
        if name in KERNELS:
            per.setdefault(name, []).append(e.device_time)
    calls = len(per.get('k_shift', []))
    out = dict((k, dict(launches=len(v), mean_us=sum(v) / len(v))) for k, v in per.items())
    out['us_per_call'] = sum(sum(v) for v in per.values()) / calls if calls else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--nx', type=int, default=126)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--freq', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_shift.py: no CUDA device (there is no CPU fallback)')
    info = card()
    runs = dict((arm_name(a), []) for a in ARMS)
    for _ in range(args.runs):
        for a in ARMS:
            runs[arm_name(a)].append(timed_run(args.nx, a, args.freq, args.steps, args.warmup))
    kernels = dict((arm_name(a), tool_kernel_us(args.nx, a, args.freq, args.profile_steps, args.warmup))
                   for a in ARMS if a is not None)
    summary = {}
    for a in ARMS:
        ms = sorted(r['ms_per_step'] for r in runs[arm_name(a)])
        summary[arm_name(a)] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_min=ms[0],
                                    ms_per_step_max=ms[-1])
    print(json.dumps(dict(workload='taylor_green_3d', integrator='PEC', nx=args.nx, steps=args.steps,
                          warmup=args.warmup, freq=args.freq, gpu=info, runs=runs,
                          summary=summary, tool_kernels=kernels, date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
