"""The cost of DensityCorrection on the flagship workload: the 3-D dam break at dx = 0.00877
(~1.22 M particles, CubicSpline, EPEC, adaptive dt, device-resident time step), one GPU.

    python bench_density_filter.py [--runs 3] [--steps 100] [--warmup 20] [--freq 10]

Three arms alternate, `runs` times each, in one process on one card: no tool, Shepard
(corr='shepard') and first-order MLS (corr='mls3d_1'), both on the fluid and the boundary every
`freq` steps, as the reference's sloshing example sets it up.  Every run builds a fresh solver,
warms up (the first filter call widens the neighbour lists there) and times `steps` steps with
CUDA events.  Reported per run: ms per step, filter calls and list builds in the timed window;
then, in a separate run of each filtering arm with torch.profiler, the mean device time of the
filter's two kernels (k_dfilter_pack + k_density_filter) per call.  The card name, power limit
and SM clock limit are read in the same process.  Prints one JSON line.  Needs a CUDA device;
writes nothing.
"""
import argparse
import json
import sys
import time

from bench_integrators import card

ARMS = (None, 'shepard', 'mls3d_1')


def make(dx, corr, freq):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    s = pb.make_wcsph_solver(pas, geo.dam_break_3d_params(dx), pb.CubicSpline(dim=3))
    tool = None
    if corr is not None:
        tool = pb.DensityCorrection(s, ['fluid', 'boundary'], corr=corr, freq=freq,
                                    kernel=pb.CubicSpline)
        s.add_tool(tool)
    return s, pas, tool


def timed_run(dx, corr, freq, steps, warmup):
    import torch
    s, pas, tool = make(dx, corr, freq)
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
    calls = 0 if tool is None else \
        sum(1 for c in range(count0, tool.count) if c % freq == 0)
    n = sum(be.sizes(i)[1] for i in range(len(pas)))
    return dict(particles=int(n), ms_per_step=e0.elapsed_time(e1) / steps, filter_calls=calls,
                list_builds=int(st['list_builds']), full_builds=int(st['full_builds']))


def filter_kernel_us(dx, corr, freq, steps, warmup):
    """device time of the filter's kernels per call, from torch.profiler (a run of its own)"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    s, _, _ = make(dx, corr, freq)
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
        if name in ('k_dfilter_pack', 'k_density_filter'):
            per.setdefault(name, []).append(e.device_time)
    calls = len(per.get('k_density_filter', []))
    out = dict((k, dict(launches=len(v), mean_us=sum(v) / len(v))) for k, v in per.items())
    out['us_per_call'] = sum(sum(v) for v in per.values()) / calls if calls else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--dx', type=float, default=0.00877)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--freq', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_density_filter.py: no CUDA device (there is no CPU fallback)')
    info = card()
    runs = dict((str(a), []) for a in ARMS)
    for _ in range(args.runs):
        for a in ARMS:
            runs[str(a)].append(timed_run(args.dx, a, args.freq, args.steps, args.warmup))
    kernels = dict((a, filter_kernel_us(args.dx, a, args.freq, args.profile_steps, args.warmup))
                   for a in ARMS if a is not None)
    summary = {}
    for a in ARMS:
        ms = sorted(r['ms_per_step'] for r in runs[str(a)])
        summary[str(a)] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_min=ms[0],
                               ms_per_step_max=ms[-1])
    print(json.dumps(dict(workload='dam_break_3d', integrator='EPEC', dx=args.dx, steps=args.steps,
                          warmup=args.warmup, freq=args.freq, gpu=info, runs=runs,
                          summary=summary, filter_kernels=kernels,
                          date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
