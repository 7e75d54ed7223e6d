"""The cost of the Interpolator on the flagship workload: the 3-D dam break at dx = 0.00877
(~1.22 M particles, CubicSpline, EPEC, adaptive dt, device-resident time step), one GPU.

    python bench_interpolator.py [--runs 3] [--steps 100] [--warmup 20] [--calls 20]

Per `interpolate('p')` call, with the Interpolator's default Gaussian kernel and 'shepard':
  * live_probes: the two obstacle probes of the reference's dam_break_3d.py:118-121 on the
    running solver;
  * live_grid: the default 125 000-point grid on the running solver;
  * private_grid: the same grid in private mode, from the state dumped to a temporary file and
    loaded back (pysph_b200.dump / load);
each timed with CUDA events around the call (the call ends with its result on the host) and
by the wall clock, `calls` calls after one warm-up call.  Then the flagship's ms per step with
a live two-point probe after every step against no probe, alternating `runs` times, each run a
fresh solver timed over `steps` steps after `warmup`.  The card name, power limit and SM clock
limit are read in the same process.  Prints one JSON line.  Needs a CUDA device; writes only
to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

from bench_integrators import card


def make(dx):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    s = pb.make_wcsph_solver(pas, geo.dam_break_3d_params(dx), pb.CubicSpline(dim=3))
    return pb, s, pas


def probes():
    # dam_break_3d.py:118-121: the obstacle's upstream face, two heights
    x_probe = 2.5 - 0.16 * 0.5
    return np.repeat(x_probe, 2), np.repeat(0.0, 2), np.array([0.021, 0.101])


def time_calls(ip, be, calls):
    import torch
    stream = torch.cuda.current_stream()
    ip.interpolate('p')
    ev, wall = [], []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record(stream)
        ip.interpolate('p')
        e1.record(stream)
        torch.cuda.synchronize()
        wall.append(1e3 * (time.perf_counter() - t0))
        ev.append(e0.elapsed_time(e1))
    ev.sort()
    wall.sort()
    return dict(points=int(np.size(ip.x)), ms_device_median=ev[len(ev) // 2], ms_device_min=ev[0],
                ms_device_max=ev[-1], ms_wall_median=wall[len(wall) // 2])


def per_call(dx, warmup, calls):
    import torch
    pb, s, pas = make(dx)
    be = s.backend
    be.use_torch_stream(torch.cuda.current_stream())
    s.initialise()
    for _ in range(warmup):
        s.step()
    out = {}
    x, y, z = probes()
    out['live_probes'] = time_calls(pb.Interpolator(pas, x=x, y=y, z=z), be, calls)
    grid = pb.Interpolator(pas)
    out['live_grid'] = time_calls(grid, be, calls)
    with tempfile.TemporaryDirectory() as tmp:
        fname = os.path.join(tmp, 'dam_break_3d_0.npz')
        s.pull()
        pb.dump(fname, pas, dict(t=0.0, dt=0.0, count=0), detailed_output=True)
        data = pb.load(fname)
    arrays = list(data['arrays'].values())
    priv = pb.Interpolator(arrays)
    priv.set_interpolation_points(grid.x, grid.y, grid.z)
    out['private_grid'] = time_calls(priv, priv._backend, calls)
    out['particles'] = int(sum(be.sizes(i)[1] for i in range(len(pas))))
    return out


def timed_run(dx, probe, steps, warmup):
    import torch
    pb, s, pas = make(dx)
    be = s.backend
    stream = torch.cuda.current_stream()
    be.use_torch_stream(stream)
    if probe:
        x, y, z = probes()
        ip = pb.Interpolator(pas, x=x, y=y, z=z)
        s.add_post_step_callback(lambda solver: ip.interpolate('p'))
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
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--dx', type=float, default=0.00877)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--calls', type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_interpolator.py: no CUDA device (there is no CPU fallback)')
    info = card()
    calls = per_call(args.dx, args.warmup, args.calls)
    runs = dict(no_probe=[], live_probe_every_step=[])
    for _ in range(args.runs):
        runs['no_probe'].append(timed_run(args.dx, False, args.steps, args.warmup))
        runs['live_probe_every_step'].append(timed_run(args.dx, True, args.steps, args.warmup))
    summary = dict((k, dict(ms_per_step_median=sorted(v)[len(v) // 2], ms_per_step_min=min(v),
                            ms_per_step_max=max(v))) for k, v in runs.items())
    print(json.dumps(dict(workload='dam_break_3d', integrator='EPEC', dx=args.dx, steps=args.steps,
                          warmup=args.warmup, gpu=info, per_call=calls, runs=runs, summary=summary,
                          date=time.strftime('%Y-%m-%d'))))


if __name__ == '__main__':
    main()
