"""ShiftPositions without a GPU: the fp64 oracle against the reference's bodies, the fixture
against its generator, the program translation and its refusals, the tool's counting, defaults
and construction-time dt, and tests/test_gpu_shift.py on the library emulation (the loader of
test_library_on_cpu.py), smaller."""
import os
import types

import numpy as np
import pytest

import test_gpu_shift as t
from helpers import load_golden
from shift_oracle import correct_velocities, shift
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)


# ---- the oracle --------------------------------------------------------------------------------
def test_oracle_matches_goldens():
    """tests/shift_oracle.py against the reference's own bodies, to 1e-12 of each particle's
    absolute sum; N_NBRS exactly."""
    for c in load_golden('shift_cases.json'):
        f = dict((k, np.array(v)) for k, v in c['inputs']['fluid'].items())
        pos = np.stack([f[k] for k in 'xyz'], axis=1)
        vel = np.stack([f[k] for k in 'uvw'], axis=1)
        L = [c['L'] if d < c['dim'] else 0.0 for d in range(3)]
        dpos, nn, scale = shift(pos, vel, f['h'], f['m'], f['rho'], c['kind'], c['const'], c['dt'],
                                c['kernel'], c['dim'], L, tensile=c['tensile'])
        want = np.array(c['dpos']).reshape(-1, 3)
        assert np.all(np.abs(dpos - want) <= 1e-12 * scale[:, None] + 1e-300), (c['kernel'], c['dim'])
        assert np.array_equal(nn, c['n_nbrs'])
        if c['correct']:
            new = t.shifted(c)
            du, nn, cs = correct_velocities(new, vel, f['h'], f['m'], f['rho'], want, c['kernel'], c['dim'], L)
            got = vel + du
            assert np.all(np.abs(got - np.stack([c[k] for k in 'uvw'], axis=1)) <=
                          1e-12 * cs[:, None] + 2 * np.spacing(np.abs(got))), (c['kernel'], c['dim'])
            assert np.array_equal(nn, c['n_nbrs_correct'])


def test_goldens_cover_the_edges():
    """An isolated particle (simple: ri = 0, dpos = 0), a particle at rest (fickian: dpos = 0),
    periodic boxes, the tensile correction, the default and a given constant, 1-3 D."""
    cases = load_golden('shift_cases.json')
    assert {(c['kernel'], c['dim']) for c in cases} == {
        (k, d) for k in ('CubicSpline', 'WendlandQuintic', 'QuinticSpline', 'Gaussian')
        for d in (1, 2, 3) if (k, d) != ('WendlandQuintic', 1)}
    assert {(c['kind'], c['correct']) for c in cases} == {
        (k, cv) for k in ('simple', 'fickian') for cv in (False, True)}
    assert any(c['tensile'] for c in cases) and any(c['L'] for c in cases)
    assert any(c['parameter'] is None for c in cases) and any(c['parameter'] for c in cases)
    for c in cases:
        dpos = np.array(c['dpos']).reshape(-1, 3)
        if c['kind'] == 'fickian':
            assert np.all(dpos[0] == 0.0)                  # at rest
        if not c['L']:
            assert c['n_nbrs'][-1] == 1                     # isolated: itself only
            if c['kind'] == 'simple':
                assert np.all(dpos[-1] == 0.0)


def test_generator_reproduces_the_fixture():
    """tests/gen_shift_golden.py, from its seeds, writes the committed cases (a sample of them,
    one per kind of geometry)."""
    gen = pytest.importorskip('gen_shift_golden')
    if not os.path.isfile(os.path.join(gen.REF, 'pysph', 'sph', 'wc', 'shift.py')):
        pytest.skip('the reference is not present')
    kernels, sh = gen.load()
    sh.sqrt = __import__('math').sqrt
    cases = load_golden('shift_cases.json')
    only = {0, 1, 2, 3, len(cases) // 2, len(cases) - 1}
    got = gen.gen_cases(kernels, sh, only=only)
    assert len(got) == len(cases)
    for i in only:
        assert got[i] == cases[i], i


# ---- program translation -------------------------------------------------------------------------
def _reference_shaped(name, **attrs):
    """an equation class of the reference's shape: same name, Python bodies"""
    def loop_all(self, d_idx, d_x, s_x, NBRS, N_NBRS):
        pass

    def __init__(self, dest, sources, **kw):
        self.dest, self.sources = dest, sources
        self.__dict__.update(attrs)
        self.__dict__.update(kw)
    return type(name, (object,), dict(__init__=__init__, loop_all=loop_all))


def test_program_translation():
    import pysph_b200 as pb
    from pysph_b200 import _lib
    from pysph_b200.program import build_program
    names = ['fluid', 'wall']
    ops = build_program([pb.Group([pb.SimpleShift('wall', ['wall'], const=0.1)], update_nnps=True),
                         pb.Group([pb.CorrectVelocities('wall', ['wall'])])], names, 2)
    assert ops == [('shift', _lib.SHIFT_SIMPLE, 2, 0.1, 1.0, 0, 0.0, 0.0), ('update_nnps',),
                   ('correct_vel', 2)]
    ops = build_program([pb.Group([pb.FickianShift('fluid', ['fluid'], fickian_const=4, hdx=1.2,
                                                    tensile_correction=True)])], names, 3)
    assert ops == [('shift', _lib.SHIFT_FICKIAN, 1, 4.0, 1.2, 1, 0.2, 4.0)]
    # the reference's own objects: recognised by class name, never handed to the generic fallback
    simple = _reference_shaped('SimpleShift', beta=0.04)
    fick = _reference_shaped('FickianShift', fickian_const=10, tensile_const=0.2, tensile_pow=4,
                             hdx=1.0, tensile_correction=False)
    cv = _reference_shaped('CorrectVelocities')
    ops = build_program([pb.Group([simple('fluid', ['fluid'])], update_nnps=True),
                         pb.Group([fick('wall', ['wall'])]), pb.Group([cv('fluid', ['fluid'])])],
                        names, 2, kernel=pb.CubicSpline(dim=2))
    assert ops == [('shift', 0, 1, 0.04, 1.0, 0, 0.0, 0.0), ('update_nnps',),
                   ('shift', 1, 2, 10.0, 1.0, 0, 0.2, 4.0), ('correct_vel', 1)]


def test_program_refusals():
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    names = ['fluid', 'wall']
    bad = [
        ([pb.SimpleShift('fluid', ['fluid']), pb.SummationDensity('wall', ['wall'])], {}, 'share a Group'),
        ([pb.SimpleShift('fluid', ['fluid']), pb.CorrectVelocities('fluid', ['fluid'])], {}, 'share a Group'),
        ([pb.FickianShift('fluid', ['fluid', 'wall'])], {}, 'only source'),
        ([pb.CorrectVelocities('fluid', ['wall'])], {}, 'only source'),
        ([pb.SimpleShift('fluid', ['fluid'])], dict(start_idx=2), 'start_idx'),
    ]
    for eqs, kw, msg in bad:
        with pytest.raises(NotImplementedError, match=msg):
            build_program([pb.Group(eqs, **kw)], names, 2)
    with pytest.raises(ValueError, match='unknown destination'):
        build_program([pb.Group([pb.SimpleShift('ghost', ['ghost'])])], names, 2)


# ---- the tool ------------------------------------------------------------------------------------
def _stub_solver(dim=2, pm=None, domain=None, dt=1e-3):
    import pysph_b200 as pb
    pa = pb.get_particle_array_wcsph(name='fluid', x=np.zeros(3))
    return types.SimpleNamespace(kernel=pb.QuinticSpline(dim=dim), pm=pm, particles=[pa], dt=dt,
                                 nnps=types.SimpleNamespace(domain=domain),
                                 backend=types.SimpleNamespace(index={'fluid': 0}))


@pytest.mark.parametrize('freq,want', [(1, [1, 2, 3, 4, 5, 6, 7]), (3, [3, 6]), (0, [])])
def test_tool_counts_steps_like_the_reference(freq, want):
    """post_step shifts after steps freq, 2 freq, ... (count starts at 1); never with freq 0"""
    import pysph_b200 as pb
    s = _stub_solver()
    tool = pb.ShiftPositions(s, 'fluid', freq=freq)
    done = []
    tool.shift = lambda: done.append(step)
    for step in range(1, 8):
        tool.post_step(s)
    assert done == want and tool.count == 8


def test_tool_defaults_and_dt():
    """the reference's signature and defaults: freq 1, simple, no correction; the constant 0.04
    (simple) or 4 (fickian, not FickianShift's own 10) unless `parameter` is truthy; dt is the
    solver's when the tool is made; vmax, dpos (and gradv) on the host array"""
    import inspect
    import pysph_b200 as pb
    sig = inspect.signature(pb.ShiftPositions.__init__)
    assert [(p.name, p.default) for p in list(sig.parameters.values())[1:]] == [
        ('app', inspect.Parameter.empty), ('array_name', inspect.Parameter.empty), ('freq', 1),
        ('shift_kind', 'simple'), ('correct_velocity', False), ('parameter', None)]
    s = _stub_solver(dt=2e-4)
    app = types.SimpleNamespace(solver=s, particles=s.particles)
    tool = pb.ShiftPositions(app, 'fluid')
    assert (tool.freq, tool.kind, tool.correct_velocity, tool.const) == (1, 'simple', False, 0.04)
    s.dt = 1.0
    assert tool.dt == 2e-4
    assert pb.ShiftPositions(app, 'fluid', shift_kind='fickian').const == 4
    assert pb.ShiftPositions(app, 'fluid', shift_kind='fickian', parameter=0).const == 4
    assert pb.ShiftPositions(app, 'fluid', parameter=0.5).const == 0.5
    assert pb.FickianShift('f', ['f']).fickian_const == 10
    pa = s.particles[0]
    assert 'vmax' in pa.constants and 'dpos' in pa.properties and 'gradv' not in pa.properties
    pb.ShiftPositions(app, 'fluid', correct_velocity=True)
    assert pa.properties['gradv'].size == 9 * 3 and pa.properties['dpos'].size == 3 * 3


def test_tool_refusals():
    import pysph_b200 as pb
    with pytest.raises(ValueError, match='shift_kind should be one of'):
        pb.ShiftPositions(_stub_solver(), 'fluid', shift_kind='fick')
    with pytest.raises(ValueError, match='no particle array'):
        pb.ShiftPositions(_stub_solver(), 'solid')
    with pytest.raises(NotImplementedError, match='slab decomposition'):
        pb.ShiftPositions(_stub_solver(pm=object()), 'fluid')
    with pytest.raises(NotImplementedError, match='mirror'):
        pb.ShiftPositions(_stub_solver(domain=pb.DomainManager(xmin=0.0, xmax=1.0, mirror_in_x=True)),
                          'fluid')
    # periodic domains are the tool's reason to be
    pb.ShiftPositions(_stub_solver(domain=pb.DomainManager(xmin=0.0, xmax=1.0, periodic_in_x=True)),
                      'fluid')


# ---- the GPU checks on the library emulation -----------------------------------------------------
@pytest.mark.parametrize('idx', list(range(0, 44, 2)))
def test_goldens_emulated(emulated_library, idx):
    t.check_goldens(idx)


@pytest.mark.parametrize('kind,correct', [('simple', False), ('fickian', True)])
def test_taylor_green_vs_oracle_emulated(emulated_library, kind, correct):
    t.check_taylor_green_vs_oracle(2, 16, kind, correct)


def test_taylor_green_3d_vs_oracle_emulated(emulated_library):
    t.check_taylor_green_vs_oracle(3, 8, 'simple', True, steps=4, freq=2)


def test_evaluation_after_shift_emulated(emulated_library):
    t.check_evaluation_after_shift(3, 8)


def test_wcsph_periodic_vs_oracle_emulated(emulated_library):
    t.check_wcsph_periodic_vs_oracle(2, 16, 'fickian', True)


def test_tvdrk3_dam_break_vs_oracle_emulated(emulated_library):
    t.check_tvdrk3_dam_break_vs_oracle(0.08, 'simple', True)


def test_lists_widen_once_emulated(emulated_library):
    t.check_lists_widen_once(dx=0.08)


def test_async_dump_at_shift_step_emulated(emulated_library, tmp_path):
    t.check_async_dump_at_shift_step(tmp_path, nx=8)


def test_refusals_on_the_library_emulated(emulated_library):
    t.check_refusals_on_the_library()
