"""ShiftPositions' particle shifting (SimpleShift, FickianShift, CorrectVelocities) on the
device: k_shift / k_correct_velocities against the reference's own bodies (shift_cases.json),
the Group route against the tool, whole periodic runs (EDAC Taylor-Green in 2-D and 3-D, a
WCSPH box under EPEC) and a dam break under TVD-RK3 against the fp64 oracle with the tool, the
evaluation right after a shift, the list widening, an asynchronous dump and the refusals.

Tolerances (per particle, against the fixture, relative to the sum of the absolute values of
the particle's terms, from tests/shift_oracle.py):
  * SimpleShift: everything is fp64 on the device; only the order of the sums differs: 1e-12.
  * FickianShift: the kernel polynomial is sph_kernel<K> in fp32 (its argument q rounded to
    fp32), everything else fp64.  The polynomial's rounding is absolute, not relative to its
    value (its pieces cancel near q = 0), and the net sum cancels strongly on a near-regular
    lattice, so the bound is stated relative to sum_j |V_j (1 + f_ij)| max|grad W(h_ij)|: 2e-6
    (the library emulation measures 1.0e-7 on the fixture).
  * CorrectVelocities: the same scale times |v_ij| |dpos_i|, where dpos carries the shift's
    own bound: 2e-5 (measured 1.7e-6).
Positions and velocities are compared with that bound plus two ulps of the value they are added
to.

The check_* functions take the sizes as arguments: tests/test_shift_on_cpu.py runs the same
checks, smaller, on the library emulation.
"""
import types

import numpy as np
import pytest

from helpers import EDAC_FIELDS, copy_arrays, load_golden, rel_err
from shift_oracle import correct_velocities, shift, with_shift

pytestmark = pytest.mark.gpu

TOL = {'simple': 1e-12, 'fickian': 2e-6, 'correct': 2e-5}
NAMES = ('fluid', 'wall')


# ---- helpers ---------------------------------------------------------------------------------
def case_arrays(case):
    import pysph_b200 as pb
    return [pb.get_particle_array_wcsph(name=n, **dict(
        (k, np.array(v, dtype=float)) for k, v in case['inputs'][n].items())) for n in NAMES]


def _domain(case):
    import pysph_b200 as pb
    if not case['L']:
        return None
    kw = {}
    for d, c in enumerate('xyz'[:case['dim']]):
        kw.update({c + 'min': 0.0, c + 'max': case['L'], 'periodic_in_' + c: True})
    return pb.DomainManager(**kw)


def _app(pas, kernel, dm, dt):
    """what ShiftPositions reads of an application: .solver (dt, kernel, backend, nnps, pm) and
    .particles"""
    import pysph_b200 as pb
    be = pb.B200Backend(pas)
    nnps = pb.B200NNPS(kernel.dim, pas, backend=be, kernel=kernel, domain=dm)
    solver = types.SimpleNamespace(dt=dt, kernel=kernel, backend=be, nnps=nnps, pm=None,
                                   particles=pas)
    return types.SimpleNamespace(solver=solver, particles=pas)


def _tool_route(case):
    import pysph_b200 as pb
    pas = case_arrays(case)
    app = _app(pas, getattr(pb, case['kernel'])(dim=case['dim']), _domain(case), case['dt'])
    tool = pb.ShiftPositions(app, 'fluid', freq=1, shift_kind=case['kind'],
                             correct_velocity=case['correct'], parameter=case['parameter'])
    tool.post_step(app.solver)
    app.solver.nnps.update_domain()      # (the Group route's update_nnps after the shift)
    app.solver.backend.pull_all()
    return pas


def _groups(case):
    import pysph_b200 as pb
    if case['kind'] == 'simple':
        eq = pb.SimpleShift('fluid', ['fluid'], const=case['const'])
    else:
        eq = pb.FickianShift('fluid', ['fluid'], fickian_const=case['const'],
                             tensile_correction=case['tensile'])
    groups = [pb.Group([eq], update_nnps=True)]
    if case['correct']:
        groups.append(pb.Group([pb.CorrectVelocities('fluid', ['fluid'])]))
    return groups


def _group_route(case):
    """B200AccelerationEval with the Groups ShiftPositions builds (shift.py:238-255); dt from
    compute(t, dt).  Returns the arrays and the accepted entries of the shift and correction."""
    import pysph_b200 as pb
    pas = case_arrays(case)
    kernel = getattr(pb, case['kernel'])(dim=case['dim'])
    ae = pb.B200AccelerationEval(pas, _groups(case), kernel)
    ae.set_nnps(pb.B200NNPS(kernel.dim, pas, backend=ae.backend, kernel=kernel, domain=_domain(case)))
    ae.count_pairs = True
    ae.compute(0.0, case['dt'])
    ae.backend.pull_all()
    return pas, ae.last_pairs


def _ulp2(a):
    return 2.0 * np.spacing(np.abs(a))


def _periodic_diff(a, b, L):
    d = a - b
    return d - L * np.round(d / L) if L else d


def shifted(case):
    """the positions the reference's body leaves: d_x += d_dpos"""
    f = case['inputs']['fluid']
    dpos = np.array(case['dpos']).reshape(-1, 3)
    return np.stack([np.array(f[c]) + dpos[:, d] for d, c in enumerate('xyz')], axis=1)


def _check_case(case, pas):
    f = dict((k, np.array(v)) for k, v in case['inputs']['fluid'].items())
    pos = np.stack([f[c] for c in 'xyz'], axis=1)
    vel = np.stack([f[c] for c in 'uvw'], axis=1)
    L = [case['L'] if d < case['dim'] else 0.0 for d in range(3)]
    _, _, scale = shift(pos, vel, f['h'], f['m'], f['rho'], case['kind'], case['const'],
                        case['dt'], case['kernel'], case['dim'], L, tensile=case['tensile'])
    fl = pas[0]
    tol = TOL[case['kind']]
    new = shifted(case)
    for d, c in enumerate('xyz'):
        err = np.abs(_periodic_diff(fl.properties[c], new[:, d], case['L']))
        bound = tol * scale + _ulp2(new[:, d])
        assert np.all(err <= bound), (c, np.max(err / bound))
    if case['correct']:
        # du is linear in dpos: the scale carries dpos's own error bound as well
        dpos = np.array(case['dpos']).reshape(-1, 3)
        _, _, cscale = correct_velocities(new, vel, f['h'], f['m'], f['rho'], dpos, case['kernel'],
                                          case['dim'], L)
        dn = np.linalg.norm(dpos, axis=1)
        cscale = cscale * np.where(dn > 0, (dn + tol * scale) / np.where(dn > 0, dn, 1.0), 0.0)
        for c in 'uvw':
            want = np.array(case[c])
            err = np.abs(fl.properties[c] - want)
            bound = TOL['correct'] * cscale + _ulp2(want)
            assert np.all(err <= bound), (c, np.max(err / bound))
    else:
        for c in 'uvw':
            assert np.array_equal(fl.properties[c], f[c])
    # the second array is never a source nor a destination (a periodic box wraps it, as any array)
    w = pas[1]
    for k, v in case['inputs']['wall'].items():
        if k in 'xyz' and case['L']:
            assert np.all(np.abs(_periodic_diff(w.properties[k], np.array(v), case['L'])) <= _ulp2(case['L'])), k
        else:
            assert np.array_equal(w.properties[k], np.array(v)), k


# ---- 1. the kernels against the reference's bodies -------------------------------------------
def check_goldens(idx=None):
    """Every case (every kernel in 1-3 D, simple and fickian, with and without the correction, a
    given and the default constant, the tensile correction, a free surface over a wall that is
    ignored, variable h, an isolated particle, a particle at rest, periodic boxes): positions and
    velocities against the reference's bodies; the accepted entries are the fixture's N_NBRS;
    the Group route is bitwise the tool route."""
    cases = load_golden('shift_cases.json')
    for c in (cases if idx is None else [cases[idx]]):
        gpas, pairs = _group_route(c)
        _check_case(c, gpas)
        assert pairs == sum(c['n_nbrs']) + sum(c.get('n_nbrs_correct', [])), (pairs, c['kernel'], c['dim'])
        if c['tensile']:
            continue                          # (the tool never sets tensile_correction)
        tpas = _tool_route(c)
        for pa, qa in zip(tpas, gpas):
            for k in ('x', 'y', 'z', 'u', 'v', 'w'):
                assert np.array_equal(pa.properties[k], qa.properties[k]), (pa.name, k)


# ---- 2. whole runs against the oracle --------------------------------------------------------
def _with_tool(s, kind, correct, freq, name='fluid'):
    import pysph_b200 as pb
    tool = pb.ShiftPositions(s, name, freq=freq, shift_kind=kind, correct_velocity=correct)
    s.add_tool(tool)
    calls = []
    run = tool.shift

    def shift_and_record():
        calls.append(s.count + 1)         # post_step runs before the solver counts the step
        run()
    tool.shift = shift_and_record
    return tool, calls


def _tg_domain(dim):
    import pysph_b200 as pb
    kw = dict(xmin=0.0, xmax=1.0, ymin=0.0, ymax=1.0, periodic_in_x=True, periodic_in_y=True)
    if dim == 3:
        kw.update(zmin=0.0, zmax=1.0, periodic_in_z=True)
    dom = ([0.0, 0.0, 0.0], [1.0, 1.0, 1.0 if dim == 3 else 0.0], [1, 1, 1 if dim == 3 else 0])
    return pb.DomainManager(**kw), dom


def _tg_solver(dim, nx, perturb, kernel='QuinticSpline'):
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from test_gpu_edac import _scheme
    pa = geo.taylor_green_particles(nx, dim=dim, perturb=perturb)
    ref = geo.taylor_green_particles(nx, dim=dim, perturb=perturb)
    p = geo.taylor_green_params(nx, dim=dim)
    dm, dom = _tg_domain(dim)
    s = pb.make_edac_solver([pa], _scheme(p, ['fluid']), getattr(pb, kernel)(dim=dim), dt=p['dt'],
                            domain=dm)
    return s, pa, ref, p, dom


def check_taylor_green_vs_oracle(dim, nx, kind, correct, steps=7, freq=3, perturb=0.2):
    """The periodic EDAC Taylor-Green (PEC + EDACTVFStep, QuinticSpline, fixed dt) with
    ShiftPositions(freq) against the oracle running the same steps: shifts after steps 3 (odd)
    and 6 (even), so both the x and the x0 buffers hold the live positions at a shift; the state
    within the bars of the unshifted Taylor-Green runs (test_gpu_edac)."""
    from oracle import oracle as orc
    s, pa, ref, p, dom = _tg_solver(dim, nx, perturb)
    tool, calls = _with_tool(s, kind, correct, freq)
    o = with_shift(orc.EDACOracleSolver)([ref], p, 'QuinticSpline', freq=freq, kind=kind,
                                          correct=correct, dt=p['dt'], domain=dom)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        s.step()
        o.step()
    assert calls == o.shifted_after == list(range(freq, steps + 1, freq)), (calls, o.shifted_after)
    s.pull()
    r = o.pas[0]
    nr = r.num_real_particles
    order = np.argsort(pa.gid)
    for f, tol in (('x', 2e-7), ('y', 2e-7), ('z', 2e-7), ('u', 5e-6), ('v', 5e-6),
                   ('w', 5e-6), ('p', 2e-5), ('rho', 2e-6)):
        want = r.properties[f][:nr]
        scale = max(np.max(np.abs(want)), 1.0 if f in 'xyz' else 1e-12)
        got = pa.properties[f][order]
        d = _periodic_diff(got, want, 1.0) if f in 'xyz' else got - want
        assert np.max(np.abs(d)) / scale <= tol, (f, np.max(np.abs(d)) / scale)


def check_evaluation_after_shift(dim, nx, kind='simple', perturb=0.2):
    """The first evaluation after a shift (the tool's NNPS update, no other) against the oracle
    evaluated on the state pulled from the device: stale packed records would show here."""
    from oracle import oracle as orc
    from test_gpu_edac import TOL as ETOL
    s, pa, _, p, dom = _tg_solver(dim, nx, perturb)
    _with_tool(s, kind, True, 1)
    s.step()
    s.nnps.update_domain()
    s.nnps.update()
    s.pull()
    from pysph_b200.particle_array import get_particle_array_edac
    n = pa.get_number_of_particles()
    opas = [get_particle_array_edac(name='fluid', **dict(
        (k, v.copy()) for k, v in pa.properties.items() if v.size == n))]   # (not dpos)
    s.a_eval.compute(s.t, p['dt'])
    s.pull()
    o = orc.EDACOracleSolver(opas, p, 'QuinticSpline', domain=dom)
    o.evaluate(s.t)
    r = o.pas[0]
    nr = r.num_real_particles
    for f in EDAC_FIELDS:
        want = r.properties[f][:nr]
        if np.max(np.abs(want)) == 0.0:
            continue
        assert rel_err(pa.properties[f], want) <= ETOL[f], f


def check_wcsph_periodic_vs_oracle(dim, n, kind, correct, steps=5, freq=2):
    """A WCSPH box periodic in every axis under EPEC (adaptive dt) with the tool against the
    oracle: the bars of test_gpu_periodic's runs."""
    import pysph_b200 as pb
    from oracle import oracle as orc
    from test_gpu_periodic import _periodic_case
    pa, params = _periodic_case(dim, n)
    ref, _ = _periodic_case(dim, n)
    kw = dict(xmin=0, xmax=1, ymin=0, ymax=1, periodic_in_x=True, periodic_in_y=True)
    if dim == 3:
        kw.update(zmin=0, zmax=1, periodic_in_z=True)
    dm = pb.DomainManager(**kw)
    s = pb.make_wcsph_solver([pa], dict(params), pb.CubicSpline(dim=dim), domain=dm)
    tool, calls = _with_tool(s, kind, correct, freq)
    dom = ([0.0] * 3, [1.0, 1.0, 1.0 if dim == 3 else 0.0], [1, 1, int(dim == 3)])
    o = with_shift(orc.WCSPHOracleSolver)([ref], dict(params), 'CubicSpline', freq=freq, kind=kind,
                                           correct=correct, dt=tool.dt, domain=dom)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        s.step()
        o.step()
    assert calls == o.shifted_after == list(range(freq, steps + 1, freq))
    s.pull()
    r = o.pas[0]
    nr = r.num_real_particles
    order = np.argsort(pa.gid)
    for k in ('x', 'y', 'z', 'u', 'v', 'w', 'rho'):
        want = r.properties[k][:nr]
        scale = max(np.max(np.abs(want)), 1e-12)
        got = pa.properties[k][order]
        d = _periodic_diff(got, want, 1.0) if k in 'xyz' else got - want
        assert np.max(np.abs(d)) <= 2e-5 * scale, k
    assert abs(s.t - o.t) <= 1e-6 * o.t


def check_tvdrk3_dam_break_vs_oracle(dx, kind, correct, steps=6, freq=3):
    """The 3-D dam break under TVD-RK3 with the tool on the fluid (the walls are no sources)
    against the oracle: the bars of the TVD-RK3 dam-break tests."""
    from pysph_b200 import geometry as geo
    from test_gpu_tvdrk3 import _compare_state, _solver
    from tvdrk3_oracle import TVDRK3OracleSolver
    pas = geo.dam_break_3d_particles(dx=dx)
    params = dict(geo.dam_break_3d_params(dx), integrator='TVDRK3')
    opas = copy_arrays(pas)
    s = _solver(pas, params)
    tool, calls = _with_tool(s, kind, correct, freq)
    o = with_shift(TVDRK3OracleSolver)(opas, params, 'CubicSpline', freq=freq, kind=kind,
                                       correct=correct, dt=tool.dt)
    s.initialise()
    o.initialise()
    for _ in range(steps):
        assert abs(s.dt - o.dt) <= 1e-6 * o.dt
        s.step()
        o.step()
    assert calls == o.shifted_after == list(range(freq, steps + 1, freq))
    s.pull()
    _compare_state(pas, opas, params)


# ---- 3. the lists widen once; a dump at a shift step -------------------------------------------
def check_lists_widen_once(dx, steps=7, freq=2):
    """The WCSPH Group's lists hold no wall-wall entries; the first shift of the walls widens
    them (one list build at most) and later calls build none.  Only calls whose own NNPS update
    kept the build are counted."""
    import pysph_b200 as pb
    from pysph_b200 import geometry as geo
    from test_gpu_tvdrk3 import _solver
    pas = geo.dam_break_3d_particles(dx=dx)
    s = _solver(pas, geo.dam_break_3d_params(dx))
    tool = pb.ShiftPositions(s, 'boundary', freq=freq, shift_kind='fickian', correct_velocity=True)
    s.add_tool(tool)
    seen = []

    def shift_counted():
        s.nnps.update_domain()
        st0 = s.backend.stats()
        s.nnps.update()
        st1 = s.backend.stats()
        s.backend.ctx.call('b200sph_shift', tool._mask, tool._kind, tool.dt, tool.const, 1.0, 0, 0.2, 4.0, None)
        s.nnps.update_domain()
        s.nnps.update()
        st2 = s.backend.stats()
        s.backend.ctx.call('b200sph_correct_velocities', tool._mask, None)
        st3 = s.backend.stats()
        if st1['full_builds'] == st0['full_builds']:
            seen.append(st1['list_builds'] - st0['list_builds'] + st2['list_builds'] - st1['list_builds'])
            seen.append(st3['list_builds'] - st2['list_builds'])
    tool.shift = shift_counted
    for _ in range(steps):
        s.step()
    assert len(seen) >= 4, seen
    assert sum(seen) <= 1, seen


def _run_tg_with_tool(steps, nx, freq, **solve):
    s, pa, _, p, _ = _tg_solver(3, nx, 0.2)
    _with_tool(s, 'fickian', True, freq)
    if solve:
        s.solve(**solve)
    for _ in range(steps):
        s.step()
    s.pull()
    return s, pa


def check_async_dump_at_shift_step(tmp_path, nx, freq=3):
    """solve(pfreq = freq) with asynchronous output: the file of a shift step holds the shifted
    positions and corrected velocities (those of a run stepped to the same count and pulled)."""
    import os
    from pysph_b200 import output
    _run_tg_with_tool(0, nx, freq, max_steps=2 * freq, pfreq=freq,
                      output_directory=str(tmp_path), asynchronous=True)
    d = output.load(os.path.join(str(tmp_path), 'b200_%05d.npz' % freq))
    _, pa = _run_tg_with_tool(freq, nx, freq)
    got = d['arrays']['fluid']
    for k in ('x', 'y', 'z', 'u', 'v', 'w'):
        assert np.array_equal(got.properties[k], pa.properties[k][:len(got.properties[k])]), k


# ---- 4. refusals ------------------------------------------------------------------------------
def check_refusals_on_the_library():
    import pysph_b200 as pb
    from pysph_b200 import _lib
    c = [k for k in load_golden('shift_cases.json') if k['dim'] == 2 and not k['L']][0]

    def setup(dm=None):
        pas = case_arrays(c)
        kernel = getattr(pb, c['kernel'])(dim=2)
        be = pb.B200Backend(pas)
        be.ctx.call('b200sph_set_kernel', 0, 2)
        pb.B200NNPS(2, pas, backend=be, kernel=kernel, domain=dm)
        return be

    be = setup()
    with pytest.raises(_lib.B200Error, match='unknown kind'):
        be.ctx.call('b200sph_shift', 1, 5, 1e-3, 0.04, 1.0, 0, 0.2, 4.0, None)
    with pytest.raises(_lib.B200Error, match='bad array mask'):
        be.ctx.call('b200sph_shift', 4, 0, 1e-3, 0.04, 1.0, 0, 0.2, 4.0, None)
    with pytest.raises(_lib.B200Error, match='no shift of the arrays'):
        be.ctx.call('b200sph_correct_velocities', 1, None)
    be.ctx.call('b200sph_shift', 1, 0, 1e-3, 0.04, 1.0, 0, 0.2, 4.0, None)
    with pytest.raises(_lib.B200Error, match='NNPS is stale'):
        be.ctx.call('b200sph_correct_velocities', 1, None)
    with pytest.raises(_lib.B200Error, match='NNPS is stale'):
        be.ctx.call('b200sph_shift', 1, 0, 1e-3, 0.04, 1.0, 0, 0.2, 4.0, None)
    be = setup(pb.DomainManager(xmin=-1.0, xmax=4.0, mirror_in_x=True))
    with pytest.raises(_lib.B200Error, match='mirror domains'):
        be.ctx.call('b200sph_shift', 1, 0, 1e-3, 0.04, 1.0, 0, 0.2, 4.0, None)


# ---- the GPU tests ----------------------------------------------------------------------------
def test_goldens(gpu_device):
    check_goldens()


@pytest.mark.parametrize('kind', ['simple', 'fickian'])
@pytest.mark.parametrize('correct', [False, True])
@pytest.mark.parametrize('dim,nx', [(2, 32), (3, 12)])
def test_taylor_green_vs_oracle(gpu_device, dim, nx, kind, correct):
    check_taylor_green_vs_oracle(dim, nx, kind, correct)


@pytest.mark.parametrize('kind', ['simple', 'fickian'])
def test_evaluation_after_shift(gpu_device, kind):
    check_evaluation_after_shift(3, 12, kind)


@pytest.mark.parametrize('kind,correct', [('simple', False), ('fickian', True)])
@pytest.mark.parametrize('dim,n', [(2, 24), (3, 10)])
def test_wcsph_periodic_vs_oracle(gpu_device, dim, n, kind, correct):
    check_wcsph_periodic_vs_oracle(dim, n, kind, correct)


@pytest.mark.parametrize('kind,correct', [('simple', True), ('fickian', False)])
def test_tvdrk3_dam_break_vs_oracle(gpu_device, kind, correct):
    check_tvdrk3_dam_break_vs_oracle(0.05, kind, correct)


def test_lists_widen_once(gpu_device):
    check_lists_widen_once(dx=0.03)


def test_async_dump_at_shift_step(gpu_device, tmp_path):
    check_async_dump_at_shift_step(tmp_path, nx=16)


def test_refusals_on_the_library(gpu_device):
    check_refusals_on_the_library()
