"""DensityCorrection without a GPU: the fp64 oracle against the reference's bodies, the program
translation and its refusals, the tool's step counting, and tests/test_gpu_density_filter.py
on the library emulation (the loader of test_library_on_cpu.py), smaller."""
import types

import numpy as np
import pytest

import test_gpu_density_filter as t
from helpers import load_golden
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

DX = 0.08


# ---- the oracle --------------------------------------------------------------------------------
def test_oracle_matches_goldens():
    """tests/density_filter_oracle.py against the reference's own bodies, to 1e-12."""
    from density_filter_oracle import density_filter
    for c in load_golden('density_filter_cases.json'):
        for pa in t.case_arrays(c):
            rhotmp = density_filter(pa, c['corr'], c['kernel'], c['dim'])
            assert np.array_equal(rhotmp, np.array(c['inputs'][pa.name]['rho']))
            want = np.array(c['rho'][pa.name])
            assert np.allclose(pa.rho, want, rtol=1e-12, atol=0.0), (c['kernel'], c['dim'], c['corr'])


def test_goldens_cover_the_early_return():
    """The isolated particle and (2-D) the line of particles with x_ij = 0 take gj_solve's early
    return: their MLS rho is the plain sum m_j W_ij."""
    from density_filter_oracle import _pairs
    from oracle import oracle as orc
    for c in load_golden('density_filter_cases.json'):
        if c['corr'] == 'shepard':
            continue
        a = dict((k, np.array(v)) for k, v in c['inputs']['fluid'].items())
        pos = np.stack([a['x'], a['y'], a['z']], axis=1)
        i, j = _pairs(pos, a['h'], orc.load().orc_kernel_radius_scale(orc.K_IDS[c['kernel']]))
        rij = np.sqrt(np.sum((pos[i] - pos[j]) ** 2, axis=1))
        w = np.array([orc.kernel_w(c['kernel'], c['dim'], r, 0.5 * (a['h'][p] + a['h'][q]))
                      for r, p, q in zip(rij, i, j)])
        plain = np.zeros(len(pos))
        np.add.at(plain, i, a['m'][j] * w)
        tail = 5 if c['dim'] == 2 else 1
        assert np.allclose(np.array(c['rho']['fluid'])[-tail:], plain[-tail:], rtol=1e-12), c['kernel']


# ---- program translation -------------------------------------------------------------------------
def _reference_shaped(name):
    """an equation class of the reference's shape: same name, Python bodies"""
    def initialize(self, d_idx, d_rho, d_rhotmp):
        d_rhotmp[d_idx] = d_rho[d_idx]

    def loop_all(self, d_idx, d_rho, d_x, s_x, s_m, s_rhotmp, SPH_KERNEL, NBRS, N_NBRS):
        d_rho[d_idx] = 0.0

    def __init__(self, dest, sources):
        self.dest, self.sources = dest, sources
    return type(name, (object,), dict(__init__=__init__, initialize=initialize, loop_all=loop_all))


def test_program_translation():
    import pysph_b200 as pb
    from pysph_b200 import _lib
    from pysph_b200.program import build_program
    names = ['fluid', 'wall', 'obstacle']
    ops = build_program([pb.Group([pb.ShepardFilter('fluid', ['fluid'])], real=False),
                         pb.Group([pb.MLSFirstOrder3D('wall', ['wall']),
                                   pb.MLSFirstOrder3D('fluid', ['fluid'])])], names, 3)
    assert ops == [('dfilter', _lib.DFILTER_SHEPARD, 1, 0), ('dfilter', _lib.DFILTER_MLS3D, 3, 1)]
    # the reference's own objects: recognised by class name, never handed to the generic fallback
    for name, mode in (('ShepardFilter', 0), ('MLSFirstOrder2D', 1), ('MLSFirstOrder3D', 2)):
        cls = _reference_shaped(name)
        ops = build_program([pb.Group([cls('wall', ['wall'])], real=False)], names, 2,
                            kernel=pb.CubicSpline(dim=2))
        assert ops == [('dfilter', mode, 2, 0)]


def test_program_refusals():
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    names = ['fluid', 'wall']
    bad = [
        ([pb.ShepardFilter('fluid', ['fluid']), pb.SummationDensity('wall', ['wall'])], {}, 'share a Group'),
        ([pb.ShepardFilter('fluid', ['fluid']), pb.MLSFirstOrder2D('wall', ['wall'])], {}, 'share a Group'),
        ([pb.ShepardFilter('fluid', ['fluid', 'wall'])], {}, 'only source'),
        ([pb.MLSFirstOrder2D('fluid', ['wall'])], {}, 'only source'),
        ([pb.ShepardFilter('fluid', ['fluid'])], dict(start_idx=2), 'start_idx'),
        ([pb.ShepardFilter('fluid', ['fluid'])], dict(stop_idx=5), 'start_idx'),
    ]
    for eqs, kw, msg in bad:
        with pytest.raises(NotImplementedError, match=msg):
            build_program([pb.Group(eqs, real=False, **kw)], names, 2)


# ---- the tool ------------------------------------------------------------------------------------
def _stub_solver(dim=3, pm=None, domain=None, kernel=None):
    import pysph_b200 as pb
    return types.SimpleNamespace(kernel=kernel or pb.CubicSpline(dim=dim), pm=pm, particles=[],
                                 nnps=types.SimpleNamespace(domain=domain),
                                 backend=types.SimpleNamespace(index={'fluid': 0}))


@pytest.mark.parametrize('freq,want', [(1, [1, 2, 3, 4, 5, 6, 7]), (3, [3, 6]), (0, [])])
def test_tool_counts_steps_like_the_reference(freq, want):
    """post_step filters after steps freq, 2 freq, ... (count starts at 1); never with freq 0"""
    import pysph_b200 as pb
    s = _stub_solver()
    s.backend.add_user_property = lambda name: 110
    tool = pb.DensityCorrection(s, ['fluid'], corr='shepard', freq=freq)
    done = []
    tool.filter = lambda: done.append(step)
    for step in range(1, 8):
        tool.post_step(s)
    assert done == want and tool.count == 8


def test_tool_refusals():
    import pysph_b200 as pb
    with pytest.raises(ValueError, match='corr should be one of'):
        pb.DensityCorrection(_stub_solver(), ['fluid'], corr='mls')
    with pytest.raises(NotImplementedError, match='dim = 2'):
        pb.DensityCorrection(_stub_solver(dim=3), ['fluid'], corr='mls2d_1')
    with pytest.raises(NotImplementedError, match='dim = 3'):
        pb.DensityCorrection(_stub_solver(dim=2), ['fluid'], corr='mls3d_1')
    with pytest.raises(NotImplementedError, match='slab decomposition'):
        pb.DensityCorrection(_stub_solver(pm=object()), ['fluid'])
    for dm in (pb.DomainManager(xmin=0.0, xmax=1.0, periodic_in_x=True),
               pb.DomainManager(xmin=0.0, xmax=1.0, mirror_in_x=True)):
        with pytest.raises(NotImplementedError, match='periodic or mirror'):
            pb.DensityCorrection(_stub_solver(domain=dm), ['fluid'])
    with pytest.raises(NotImplementedError, match='radius scale'):
        pb.DensityCorrection(_stub_solver(), ['fluid'], kernel=pb.QuinticSpline)


def test_add_tool_registers_what_a_tool_overloads():
    import pysph_b200 as pb
    s = types.SimpleNamespace(pre_step_callbacks=[], post_step_callbacks=[], tools=[],
                              post_stage_callbacks=[])
    s.add_pre_step_callback = s.pre_step_callbacks.append
    s.add_post_step_callback = s.post_step_callbacks.append
    s.add_post_stage_callback = s.post_stage_callbacks.append

    class Only(pb.Tool):
        def post_step(self, solver):
            pass
    tool = Only()
    pb.B200Solver.add_tool(s, tool)
    assert s.post_step_callbacks == [tool.post_step] and not s.pre_step_callbacks
    assert not s.post_stage_callbacks and s.tools == [tool]


# ---- the GPU checks on the library emulation -----------------------------------------------------
@pytest.mark.parametrize('idx', list(range(16)))
def test_goldens_emulated(emulated_library, idx):
    t.check_goldens(idx)


@pytest.mark.parametrize('dim,integrator,corr', [(3, 'EPEC', 'shepard'), (3, 'EPEC', 'mls3d_1'),
                                                 (3, 'TVDRK3', 'shepard'), (3, 'TVDRK3', 'mls3d_1'),
                                                 (2, 'EPEC', 'mls2d_1')])
def test_dam_break_vs_oracle_emulated(emulated_library, dim, integrator, corr):
    t.check_dam_break_vs_oracle(dim, integrator, corr, dx=DX if dim == 3 else 0.06, steps=20)


@pytest.mark.parametrize('records', ['32', '48'])
@pytest.mark.parametrize('device_dt', [True, False])
def test_fused_is_bitwise_unfused_emulated(emulated_library, monkeypatch, records, device_dt):
    t.check_fused_is_bitwise_unfused(monkeypatch, records, device_dt, dx=DX, steps=10)


def test_next_evaluation_sees_filtered_rho_emulated(emulated_library):
    t.check_next_evaluation_sees_filtered_rho(dx=DX)


def test_async_dump_at_filter_step_emulated(emulated_library, tmp_path):
    t.check_async_dump_at_filter_step(tmp_path, dx=DX)


def test_lists_widen_once_emulated(emulated_library):
    t.check_lists_widen_once(dx=DX)


def test_refusals_on_the_library_emulated(emulated_library):
    t.check_refusals_on_the_library()


def test_lists_required_emulated(emulated_library, monkeypatch):
    t.check_lists_required(monkeypatch)
