"""DensityCorrection's density re-initialisation (ShepardFilter, MLSFirstOrder2D,
MLSFirstOrder3D) on the device: k_density_filter against the reference's own bodies
(density_filter_cases.json), the Group route against the tool, whole dam-break runs against
the fp64 oracle with the tool, fused against unfused, the asynchronous dump, the list widening
and the refusals.

The check_* functions take the sizes as arguments: tests/test_density_filter_on_cpu.py runs
the same checks, smaller, on the library emulation.
"""
import types

import numpy as np
import pytest

from helpers import copy_arrays, load_golden
from density_filter_oracle import with_density_correction
from test_gpu_tvdrk3 import _compare_state, _solver
from tvdrk3_oracle import TVDRK3OracleSolver

pytestmark = pytest.mark.gpu

FILTER_CLASS = {'shepard': 'ShepardFilter', 'mls2d_1': 'MLSFirstOrder2D',
                'mls3d_1': 'MLSFirstOrder3D'}
NAMES = ('fluid', 'wall')


# ---- helpers ---------------------------------------------------------------------------------
def case_arrays(case):
    import pysph_b200 as pb
    pas = []
    for name in NAMES:
        props = dict((k, np.array(v, dtype=float)) for k, v in case['inputs'][name].items())
        pa = pb.get_particle_array_wcsph(name=name, **props)
        pa.add_property('rhotmp')
        pas.append(pa)
    return pas


def _app(pas, kernel):
    """what DensityCorrection reads of an application: .solver (kernel, backend, nnps, pm) and
    .particles"""
    import pysph_b200 as pb
    be = pb.B200Backend(pas)
    nnps = pb.B200NNPS(kernel.dim, pas, backend=be, kernel=kernel)
    solver = types.SimpleNamespace(kernel=kernel, backend=be, nnps=nnps, pm=None, particles=pas)
    return types.SimpleNamespace(solver=solver, particles=pas)


def _tool_route(case):
    import pysph_b200 as pb
    pas = case_arrays(case)
    kcls = getattr(pb, case['kernel'])
    app = _app(pas, kcls(dim=case['dim']))
    tool = pb.DensityCorrection(app, list(NAMES), corr=case['corr'], freq=1, kernel=kcls)
    tool.post_step(app.solver)
    app.solver.backend.pull_all()
    return pas


def _group_route(case):
    """B200AccelerationEval with the Groups DensityCorrection builds (tools.py:133-188): one
    Group([Filter(a, [a])], real=False) per array"""
    import pysph_b200 as pb
    pas = case_arrays(case)
    kernel = getattr(pb, case['kernel'])(dim=case['dim'])
    cls = getattr(pb, FILTER_CLASS[case['corr']])
    groups = [pb.Group([cls(n, [n])], real=False) for n in NAMES]
    ae = pb.B200AccelerationEval(pas, groups, kernel)
    ae.set_nnps(pb.B200NNPS(kernel.dim, pas, backend=ae.backend, kernel=kernel))
    ae.compute(0.0, 0.0)
    ae.backend.pull_all()
    return pas


# ---- 1. the kernel against the reference's bodies --------------------------------------------
def check_goldens(idx=None, rtol=2e-6):
    """Device rho against the reference's bodies for every case (every kernel, 2-D and 3-D,
    variable h, a free surface over a wall, an isolated particle, a collinear neighbourhood);
    rhotmp is the rho from before, bitwise; the Group route is bitwise the tool route."""
    cases = load_golden('density_filter_cases.json')
    for c in (cases if idx is None else [cases[idx]]):
        pas = _tool_route(c)
        for pa in pas:
            want = np.array(c['rho'][pa.name])
            assert np.allclose(pa.rho, want, rtol=rtol, atol=0.0), \
                (c['kernel'], c['dim'], c['corr'], pa.name, np.max(np.abs(pa.rho / want - 1)))
            assert np.array_equal(pa.rhotmp, np.array(c['inputs'][pa.name]['rho']))
        for pa, qa in zip(pas, _group_route(c)):
            assert np.array_equal(pa.rho, qa.rho) and np.array_equal(pa.rhotmp, qa.rhotmp)


# ---- 2. whole runs against the oracle --------------------------------------------------------
def _with_tool(s, names, corr, freq, kcls):
    import pysph_b200 as pb
    tool = pb.DensityCorrection(s, names, corr=corr, freq=freq, kernel=kcls)
    s.add_tool(tool)
    calls = []
    run = tool.filter

    def filter_and_record():
        calls.append(s.count + 1)         # post_step runs before the solver counts the step
        run()
    tool.filter = filter_and_record
    return tool, calls


def check_dam_break_vs_oracle(dim, integrator, corr, dx, steps, freq=5, threads=4):
    """Adaptive steps of the dam break with DensityCorrection(freq) against the oracle solver
    running the same sequence: the filter after the same steps, the same dt sequence to 1e-6,
    positions and velocities within the bars of the dam-break tests.  rho: the filter's sums
    are fp32, so the filtered rho carries their rounding -- 2e-6 relative for Shepard, the
    tolerance of the SummationDensity parity, where the unfiltered runs hold 2e-7; 1e-5 for
    MLS, whose solve amplifies the rounding of the fp32 moments by the condition of A, large
    where the support is cut off in a corner of the tank."""
    rho = 2e-6 if corr == 'shepard' else 1e-5
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from oracle.oracle import WCSPHOracleSolver
    if dim == 3:
        pas = geo.dam_break_3d_particles(dx=dx)
        params, kname, names = geo.dam_break_3d_params(dx), 'CubicSpline', ['fluid', 'boundary']
    else:
        pas = geo.dam_break_2d_particles(dx=dx)
        params, kname, names = geo.dam_break_2d_params(dx=dx), 'WendlandQuintic', ['fluid', 'boundary']
    params = dict(params, integrator=integrator)
    opas = copy_arrays(pas)
    s = _solver(pas, params, kname)
    tool, calls = _with_tool(s, names, corr, freq, getattr(pb, kname))
    base = TVDRK3OracleSolver if integrator == 'TVDRK3' else WCSPHOracleSolver
    o = with_density_correction(base)(opas, params, kname, threads=threads, names=names,
                                      corr=corr, freq=freq)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        assert abs(s.dt - o.dt) <= 1e-6 * o.dt
        s.step()
        o.step()
    assert calls == o.filtered_after == list(range(freq, steps + 1, freq)), (calls, o.filtered_after)
    assert abs(s.dt - o.dt) <= 1e-6 * o.dt and abs(s.t - o.t) <= 1e-6 * o.t
    s.pull()
    _compare_state(pas, opas, params, rho=rho)


# ---- 3. fused == unfused, bitwise; the next evaluation sees the filtered rho ------------------
def _run_with_tool(dx, steps, corr='mls3d_1', freq=5, integrator='EPEC', **kw):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    rs = np.random.RandomState(4)
    pas[0].rho[:] *= 1 + 0.01 * rs.uniform(-1, 1, pas[0].rho.size)
    params = dict(geo.dam_break_3d_params(dx), integrator=integrator, n_damp=4)
    s = _solver(pas, params, **kw)
    tool, calls = _with_tool(s, ['fluid', 'boundary'], corr, freq, pb.CubicSpline)
    for _ in range(steps):
        s.step()
    st = s.backend.stats()
    s.pull()
    return s, pas, st, calls


def check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx, steps=12):
    """With the tool, the fused stage kernels against B200SPH_FUSE=0: every pullable property,
    t and dt bitwise, for 32- and 48-byte records and host and device dt."""
    if records == '48':
        monkeypatch.setenv('B200SPH_RECORDS', '48')
    else:
        monkeypatch.delenv('B200SPH_RECORDS', raising=False)
    out = {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('B200SPH_FUSE', fuse)
        s, pas, st, calls = _run_with_tool(dx, steps, device_dt=device_dt)
        assert calls == list(range(5, steps + 1, 5))
        assert (st['fused_stages'] > 0) == (fuse == '1'), st
        if fuse == '1' and records != '48':
            assert st['pair_launches_r32'] > 0, st
        out[fuse] = (s.t, s.dt, [dict((k, v.copy()) for k, v in pa.properties.items()) for pa in pas])
    a, b = out['1'], out['0']
    assert a[:2] == b[:2], (a[:2], b[:2])
    for pa, pb_ in zip(a[2], b[2]):
        for k, v in pa.items():
            assert np.array_equal(v, pb_[k]), k


def check_next_evaluation_sees_filtered_rho(dx, freq=3):
    """After a filter step the next evaluation's p is the Tait EOS of the FILTERED rho (the
    records and the speculative EOS of the fused stage were made from the rho before)."""
    from pysph_b200 import geometry as geo
    s, pas, st, calls = _run_with_tool(dx, freq, corr='shepard', freq=freq)
    assert calls == [freq]
    f = pas[0]
    rho_f, rho_before = f.rho.copy(), f.rhotmp.copy()
    assert np.max(np.abs(rho_f - rho_before)) > 1e-3 * np.max(rho_f)
    s.a_eval.compute(s.t, s.dt)            # the tool has just updated the NNPS
    s.pull()
    p = geo.dam_break_3d_params(dx)
    B = p['rho0'] * p['c0'] ** 2 / p['gamma']
    want = B * ((rho_f / p['rho0']) ** p['gamma'] - 1.0)
    scale = np.max(np.abs(want))
    assert np.max(np.abs(f.p - want)) <= 1e-5 * scale
    stale = B * ((rho_before / p['rho0']) ** p['gamma'] - 1.0)
    assert np.max(np.abs(f.p - stale)) > 1e-3 * scale


# ---- 4. a dump at a filter step --------------------------------------------------------------
def check_async_dump_at_filter_step(tmp_path, dx, freq=4):
    """solve(pfreq = freq) with asynchronous output: the file of a filter step holds the
    filtered rho (that of a run stepped to the same count and pulled)."""
    import os
    from pysph_b200 import output
    s, pas, st, calls = _run_with_tool(dx, 0, corr='mls3d_1', freq=freq)
    s.solve(max_steps=2 * freq, pfreq=freq, output_directory=str(tmp_path), asynchronous=True)
    d = output.load(os.path.join(str(tmp_path), 'b200_%05d.npz' % freq))
    _, pas_ref, _, calls_ref = _run_with_tool(dx, freq, corr='mls3d_1', freq=freq)
    assert calls[:1] == calls_ref == [freq]
    for pa in pas_ref:
        got = d['arrays'][pa.name].rho
        assert np.array_equal(got, pa.rho[:len(got)]), pa.name


# ---- 5. the lists widen once -----------------------------------------------------------------
def check_lists_widen_once(dx, steps=9, freq=2):
    """The WCSPH Group's lists hold no wall-wall entries; the first filter call of the walls
    widens them (one list build at most) and later calls build none.  Only calls whose own NNPS
    update kept the build are counted."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    pas = geo.dam_break_3d_particles(dx=dx)
    s = _solver(pas, geo.dam_break_3d_params(dx))
    tool = pb.DensityCorrection(s, ['fluid', 'boundary'], corr='shepard', freq=freq)
    s.add_tool(tool)
    seen = []

    def filter_counted():
        st0 = s.backend.stats()
        s.nnps.update_domain()
        s.nnps.update()
        st1 = s.backend.stats()
        s.backend.ctx.call('b200sph_density_filter', tool._mask, 0, tool._kid, tool._rhotmp, 0)
        st2 = s.backend.stats()
        if st1['full_builds'] == st0['full_builds']:
            seen.append(st2['list_builds'] - st1['list_builds'])
    tool.filter = filter_counted
    for _ in range(steps):
        s.step()
    assert len(seen) >= 3, seen
    assert seen[0] <= 1 and all(x == 0 for x in seen[1:]), seen


# ---- 6. refusals ------------------------------------------------------------------------------
def check_refusals_on_the_library():
    import pysph_b200 as pb
    from pysph_b200 import _lib
    c = load_golden('density_filter_cases.json')
    by = dict(((k['kernel'], k['dim'], k['corr']), k) for k in c)

    def setup(key, kernel=None, **nnps_kw):
        pas = case_arrays(by[key])
        kernel = kernel or getattr(pb, key[0])(dim=key[1])
        be = pb.B200Backend(pas)
        pb.B200NNPS(kernel.dim, pas, backend=be, kernel=kernel, **nnps_kw)
        return be, be.add_user_property('rhotmp')

    be, pid = setup(('CubicSpline', 3, 'shepard'))
    for mode, kid, msg in ((_lib.DFILTER_MLS2D, 0, 'MLSFirstOrder2D needs dim = 2'),
                           (_lib.DFILTER_SHEPARD, 2, 'radius scale'),
                           (7, 0, 'unknown mode')):
        with pytest.raises(_lib.B200Error, match=msg):
            be.ctx.call('b200sph_density_filter', 1, mode, kid, pid, 0)
    with pytest.raises(_lib.B200Error, match='user property'):
        be.ctx.call('b200sph_density_filter', 1, 0, 0, pid + 1, 0)
    with pytest.raises(_lib.B200Error, match='bad array mask'):
        be.ctx.call('b200sph_density_filter', 4, 0, 0, pid, 0)
    be, pid = setup(('CubicSpline', 2, 'shepard'))
    with pytest.raises(_lib.B200Error, match='MLSFirstOrder3D needs dim = 3'):
        be.ctx.call('b200sph_density_filter', 1, _lib.DFILTER_MLS3D, 0, pid, 0)
    for dm in (pb.DomainManager(xmin=-1.0, xmax=4.0, periodic_in_x=True),
               pb.DomainManager(xmin=-1.0, xmax=4.0, mirror_in_x=True)):
        be, pid = setup(('CubicSpline', 2, 'shepard'), domain=dm)
        with pytest.raises(_lib.B200Error, match='periodic and mirror'):
            be.ctx.call('b200sph_density_filter', 1, 0, 0, pid, 0)


def check_lists_required(monkeypatch):
    import pysph_b200 as pb
    from pysph_b200 import _lib
    monkeypatch.setenv('B200SPH_PAIR_KERNEL', 'warp')
    c = load_golden('density_filter_cases.json')[0]
    pas = case_arrays(c)
    be = pb.B200Backend(pas)
    pb.B200NNPS(c['dim'], pas, backend=be, kernel=getattr(pb, c['kernel'])(dim=c['dim']))
    pid = be.add_user_property('rhotmp')
    with pytest.raises(_lib.B200Error, match='cannot index the particles'):
        be.ctx.call('b200sph_density_filter', 1, 0, 0, pid, 0)


# ---- the GPU tests ----------------------------------------------------------------------------
def test_goldens(gpu_device):
    check_goldens()


@pytest.mark.parametrize('dim,integrator,corr', [(3, 'EPEC', 'shepard'), (3, 'EPEC', 'mls3d_1'),
                                                 (3, 'TVDRK3', 'shepard'), (3, 'TVDRK3', 'mls3d_1'),
                                                 (2, 'EPEC', 'mls2d_1')])
def test_dam_break_vs_oracle(gpu_device, dim, integrator, corr):
    check_dam_break_vs_oracle(dim, integrator, corr, dx=0.05 if dim == 3 else 0.03, steps=20)


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_fused_is_bitwise_unfused(gpu_device, monkeypatch, records, device_dt):
    check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx=0.03, steps=12)


def test_next_evaluation_sees_filtered_rho(gpu_device):
    check_next_evaluation_sees_filtered_rho(dx=0.03)


def test_async_dump_at_filter_step(gpu_device, tmp_path):
    check_async_dump_at_filter_step(tmp_path, dx=0.03)


def test_lists_widen_once(gpu_device):
    check_lists_widen_once(dx=0.03)


def test_refusals_on_the_library(gpu_device):
    check_refusals_on_the_library()


def test_lists_required(gpu_device, monkeypatch):
    check_lists_required(monkeypatch)
