"""EPEC against TVD-RK3 on the flagship workload: the 3-D dam break at dx = 0.00877
(~1.22 M particles, CubicSpline, adaptive dt, device-resident time step), one GPU.

    python bench_integrators.py [--runs 3] [--steps 100] [--warmup 20] [--dx 0.00877]

The two integrators alternate, `runs` times each, in one process on one card; every run
builds a fresh solver, warms up and times `steps` steps with CUDA events.  Reported per run:
ms per step, ms per evaluation (EPEC evaluates twice per step, TVD-RK3 three times), pairs per
second, kernel launches per step and list builds; then, in a separate run with torch.profiler,
the mean time of the fused stage kernel (k_stage_pack / k_stage_pack_rk3).  The card name,
power limit and SM clock limit are read in the same process.  Prints one JSON line.  Needs a
CUDA device; writes nothing.
"""
import argparse
import json
import subprocess
import sys
import time

INTEGRATORS = (('EPEC', 2, 'k_stage_pack'), ('TVDRK3', 3, 'k_stage_pack_rk3'))


def card():
    q = 'name,power.limit,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader'],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    return dict(zip(q.split(','), [v.strip() for v in out.splitlines()[0].split(',')]))


def make(dx, integrator):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    params = dict(geo.dam_break_3d_params(dx), integrator=integrator)
    s = pb.make_wcsph_solver(pas, params, pb.CubicSpline(dim=3))
    return s, pas


def pairs_of_one_step(s):
    """one untimed step with the pair counter on: the pairs of all its evaluations"""
    total = [0]
    integ = s.integrator
    orig = integ.compute_accelerations

    def counting(*a, **kw):
        orig(*a, **kw)
        total[0] += s.a_eval.last_pairs
    s.a_eval.count_pairs = True
    integ.compute_accelerations = counting
    s.step()
    del integ.compute_accelerations
    s.a_eval.count_pairs = False
    return total[0]


def timed_run(dx, integrator, n_eval, steps, warmup):
    import torch
    s, pas = make(dx, integrator)
    be = s.backend
    stream = torch.cuda.current_stream()
    be.use_torch_stream(stream)
    s.initialise()
    for _ in range(warmup):
        s.step()
    pairs = pairs_of_one_step(s)
    be.ctx.call('b200sph_reset_stats')
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        s.step()
    e1.record(stream)
    torch.cuda.synchronize()
    st = be.stats()
    ms = e0.elapsed_time(e1) / steps
    n = sum(be.sizes(i)[1] for i in range(len(pas)))
    return dict(particles=int(n), ms_per_step=ms, ms_per_evaluation=ms / n_eval,
                pairs_per_s=pairs / (ms * 1e-3), launches_per_step=st['kernel_launches'] / steps,
                list_builds=int(st['list_builds']), full_builds=int(st['full_builds']),
                fused_stages_per_step=st['fused_stages'] / steps)


def stage_kernel_ms(dx, integrator, name, steps, warmup):
    """mean device time of the fused stage kernel, from torch.profiler (a run of its own)"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    s, _ = make(dx, integrator)
    s.backend.use_torch_stream(torch.cuda.current_stream())
    s.initialise()
    for _ in range(warmup):
        s.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            s.step()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and e.name.split('(')[0] == name]
    return dict(kernel=name, launches=len(times),
                mean_us=(sum(times) / len(times)) if times else None)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--dx', type=float, default=0.00877)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--profile-steps', type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_integrators.py: no CUDA device (there is no CPU fallback)')
    info = card()
    runs = dict((name, []) for name, _, _ in INTEGRATORS)
    for _ in range(args.runs):
        for name, n_eval, _ in INTEGRATORS:
            runs[name].append(timed_run(args.dx, name, n_eval, args.steps, args.warmup))
    kernels = dict((name, stage_kernel_ms(args.dx, name, kname, args.profile_steps, args.warmup))
                   for name, _, kname in INTEGRATORS)
    summary = {}
    for name, _, _ in INTEGRATORS:
        ms = sorted(r['ms_per_step'] for r in runs[name])
        summary[name] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_min=ms[0],
                             ms_per_step_max=ms[-1])
    ratio = summary['TVDRK3']['ms_per_step_median'] / summary['EPEC']['ms_per_step_median']
    print(json.dumps(dict(workload='dam_break_3d', dx=args.dx, steps=args.steps,
                          warmup=args.warmup, gpu=info, runs=runs, summary=summary,
                          tvdrk3_over_epec_ms_per_step=ratio, fused_stage_kernel=kernels,
                          date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
