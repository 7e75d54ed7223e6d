"""Pin the fp64 CPU oracle against the reference (CPU only, no GPU).

Sources of truth, all generated from / stated by the reference itself:
* tests/golden/*.json  -- outputs of the reference's own compiled kernels
  (c_kernels.pyx) and its own Python equation / stepper bodies, produced by
  oracle/gen_golden.py in the build container;
* known answers hard-coded in the reference's tests (cited per test).
"""
import math

import numpy as np
import pytest

from helpers import (ACC_FIELDS, arrays_from_dict, load_golden, rel_err,
                     wcsph_params_from_case)
from oracle import oracle as orc
from pysph_b200.particle_array import get_particle_array_wcsph


# ---------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------
def test_kernels_match_reference_compiled_kernels():
    for entry in load_golden('kernels.json'):
        name, dim = entry['kernel'], entry['dim']
        kid = orc.K_IDS[name]
        lib = orc.load()
        assert lib.orc_kernel_radius_scale(kid) == entry['radius_scale']
        assert lib.orc_kernel_deltap(kid) == entry['deltap']
        for c in entry['cases']:
            scale_w = entry['fac'] / c['h'] ** dim
            w = orc.kernel_w(name, dim, c['rij'], c['h'])
            g = orc.kernel_grad(name, dim, c['xij'], c['rij'], c['h'])
            assert abs(w - c['w']) <= 1e-12 * scale_w, (name, dim, c)
            assert np.allclose(g, c['grad'], rtol=1e-11,
                               atol=1e-12 * scale_w / c['h']), (name, dim, c)


@pytest.mark.parametrize('name,dim,w0', [
    # pysph/base/tests/test_kernel.py:148,191,229,343,350,357,435,446
    ('CubicSpline', 1, 2. / 3), ('CubicSpline', 2, 10. / (7 * math.pi)),
    ('CubicSpline', 3, 1. / math.pi),
    ('QuinticSpline', 1, 0.55), ('QuinticSpline', 2, 66. * 7 / (478 * math.pi)),
    ('QuinticSpline', 3, 66. / (120 * math.pi)),
    ('WendlandQuintic', 2, 7. / (4 * math.pi)),
    ('WendlandQuintic', 3, 21. / (16 * math.pi)),
])
def test_kernel_value_at_origin(name, dim, w0):
    assert abs(orc.kernel_w(name, dim, 0.0, 1.0) - w0) < 1e-14


def test_kernel_moments_3d_cubic_spline():
    # test_kernel.py:63-113: int W = 1, int x grad W = -1 (quadrature on a grid)
    n = 41
    xs = np.linspace(-2.0, 2.0, n)
    dv = (xs[1] - xs[0]) ** 3
    m0 = 0.0
    gx = 0.0
    for x in xs:
        for y in xs:
            for z in xs:
                r = math.sqrt(x * x + y * y + z * z)
                m0 += orc.kernel_w('CubicSpline', 3, r, 1.0)
                # xij = x_i - x_j with the source at (x, y, z) and dest at 0;
                # test_kernel.py:108-113: int (x_j - x_i) dW_i/dx = 1
                gx += x * orc.kernel_grad('CubicSpline', 3, [-x, -y, -z], r, 1.0)[0]
    assert abs(m0 * dv - 1.0) < 5e-3
    assert abs(gx * dv - 1.0) < 2e-2


# ---------------------------------------------------------------------------
# no-source equations and steppers vs the reference's Python bodies
# ---------------------------------------------------------------------------
def test_eos_and_ferrari_match_reference_bodies():
    g = load_golden('eos.json')
    for name, hg in (('TaitEOS', 0), ('TaitEOSHGCorrection', 1)):
        e = g[name]
        pa = get_particle_array_wcsph(name='f', x=np.zeros(len(e['rho_in'])),
                                      rho=np.array(e['rho_in']))
        o = orc.Oracle([pa], 3)
        o.eos(0, hg, e['rho0'], e['c0'], e['gamma'], e['p0'])
        assert np.array_equal(pa.rho, e['rho_out'])
        assert np.allclose(pa.p, e['p'], rtol=1e-13, atol=1e-9)
        assert np.allclose(pa.cs, e['cs'], rtol=1e-14)
    e = g['UpdateSmoothingLengthFerrari']
    pa = get_particle_array_wcsph(name='f', x=np.zeros(len(e['rho'])),
                                  rho=np.array(e['rho']), m=np.array(e['m']))
    o = orc.Oracle([pa], 2)
    o.ferrari_h(0, e['hdx'], e['dim'])
    assert np.allclose(pa.h, e['h'], rtol=1e-14)


def test_appendix_d_known_answers():
    # SURVEY.md Appendix D2 (generated from the reference's Python bodies)
    pa = get_particle_array_wcsph(name='f', x=np.zeros(3),
                                  rho=np.array([1005.0, 998.0, 990.0]))
    o = orc.Oracle([pa], 3)
    o.eos(0, 0, 1000.0, 32.85, 7.0, 0.0)
    assert abs(pa.p[0] - 5477.224521454092) < 1e-8
    assert abs(pa.cs[0] - 33.34521785625001) < 1e-11
    assert abs(pa.p[1] - -2145.3386086737232) < 1e-8
    pa.rho[2] = 990.0
    o.eos(0, 1, 1000.0, 32.85, 7.0, 0.0)
    assert pa.rho[2] == 1000.0 and pa.p[2] == 0.0 and abs(pa.cs[2] - 32.85) < 1e-13
    # kernel values of the D2 pair
    xij = [0 - 0.011, 0 + 0.004, 0 - 0.007]
    rij = math.sqrt(sum(v * v for v in xij))
    hij = 0.5 * (0.013 + 0.0125)
    assert abs(orc.kernel_w('CubicSpline', 3, rij, hij) - 30915.966589680047) < 1e-7
    g = orc.kernel_grad('CubicSpline', 3, xij, rij, hij)
    # Appendix D quotes DWIJ for x_ij = d - s
    assert np.allclose(np.abs(g), [6306509.143779232, 2293276.0522833574,
                                   4013233.0914958753], rtol=1e-12)
    assert abs(orc.kernel_w('WendlandQuintic', 3, rij, hij) - 29627.78481739429) < 1e-7
    assert abs(orc.kernel_w('QuinticSpline', 3, rij, hij) - 28949.19091885566) < 1e-7


def test_wcsph_step_matches_reference_bodies():
    g = load_golden('steppers.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        pa = get_particle_array_wcsph(name='f', **props)
        o = orc.Oracle([pa], 3)
        o.stage(0, which, g['dt'])
        for k, v in g['outputs'][key].items():
            assert np.allclose(pa.properties[k], v, rtol=1e-15, atol=0), (key, k)


# ---------------------------------------------------------------------------
# whole evaluations vs the reference's bodies driven pair by pair
# ---------------------------------------------------------------------------
def test_density_1d_fixture():
    # pysph/sph/tests/test_acceleration_eval.py:294-303,341,737-741,760-764
    g = load_golden('density_1d.json')
    assert g['nbr_counts'] == [3, 4, 5, 5, 5, 5, 5, 5, 4, 3]
    expect = np.array([7.357] + [9.0] * 8 + [7.357])
    assert np.allclose(g['rho'], expect, atol=1e-2)
    pa = get_particle_array_wcsph(name='fluid', x=np.array(g['x']),
                                  h=np.array(g['h']), m=np.array(g['m']))
    o = orc.Oracle([pa], 1, 'CubicSpline')
    o.update_domain()
    o.nnps_update()
    pairs = o.pair_pass([(orc.EQ_SUMDENS, 0, [0])])
    assert pairs == sum(g['nbr_counts'])
    assert [len(o.neighbors(0, 0, i)) for i in range(10)] == g['nbr_counts']
    assert np.allclose(pa.rho, g['rho'], rtol=1e-14)


def run_oracle_case(case):
    pas = arrays_from_dict(case['inputs'])
    s = orc.WCSPHOracleSolver(pas, wcsph_params_from_case(case), case['kernel'])
    s.evaluate()
    return pas


@pytest.mark.parametrize('idx', range(6))
def test_wcsph_evaluation_matches_reference_bodies(idx):
    case = load_golden('wcsph_cases.json')[idx]
    pas = run_oracle_case(case)
    for pa in pas:
        ref = case['outputs'][pa.name]
        n_real = ref['_n_real']
        for f in ACC_FIELDS + ['rho', 'p', 'cs']:
            got = pa.properties[f]
            want = np.array(ref[f])
            scale = max(np.max(np.abs(want)), 1e-300)
            # identical arithmetic, only the neighbour visiting order differs
            assert np.max(np.abs(got - want)) <= 2e-12 * scale, (pa.name, f)
        assert pa.num_real_particles == n_real


# ---------------------------------------------------------------------------
# NNPS: linked list == brute force (pysph/base/tests/test_nnps.py)
# ---------------------------------------------------------------------------
def _random_arrays(seed=123):
    # test_nnps.py:303-376: seeded uniform points in [-1,1]^3, h = 1.2 dx
    rs = np.random.RandomState(seed)
    out = []
    for name, n, hv in (('a', 2048, 0.0), ('b', 1024, 0.0), ('c', 1024, 1.0)):
        x, y, z = (rs.uniform(-1, 1, n) for _ in range(3))
        dx = 2.0 / n ** (1. / 3)
        h = np.full(n, 1.2 * dx) * (1.0 + hv * rs.uniform(0, 1, n))
        out.append(get_particle_array_wcsph(name=name, x=x, y=y, z=z, h=h))
    return out


def test_linked_list_equals_brute_force():
    pas = _random_arrays()
    o = orc.Oracle(pas, 3, 'CubicSpline')
    o.update_domain()
    o.nnps_update()
    rs = np.random.RandomState(0)
    for dst in range(3):
        for src in range(3):
            n = pas[dst].get_number_of_particles()
            for i in rs.randint(0, n, 25):
                a = np.sort(o.neighbors(dst, src, i))
                b = np.sort(o.brute_neighbors(dst, src, i))
                assert np.array_equal(a, b)


def test_binning_fixture():
    # test_nnps.py:33-140: 10 hand-placed points, cell_size = 1 when h = 0
    x = np.array([0.3, 0.6, 0.1, 0.3, 0.6, 0.5, -0.3, 0.7, 0.1, 0.7])
    cells = [(-2, 0, 0), (0, -1, 0), (1, -2, 1), (0, 1, -1), (-1, 0, -2),
             (-1, 0, -2), (-2, 0, 0), (0, 1, -1), (0, -1, 0), (0, 1, -1)]
    c = np.array(cells, dtype=float)
    pa = get_particle_array_wcsph(name='a', x=c[:, 0] + x * 0.9,
                                  y=c[:, 1] + 0.5, z=c[:, 2] + 0.5,
                                  h=np.zeros(10))
    o = orc.Oracle([pa], 3, 'CubicSpline')
    o.update_domain()
    o.nnps_update()
    g = o.grid()
    assert g['cell_size'] == 1.0          # nnps_base.pyx:972-973
    # particles sharing a cell in the fixture share a cell here
    ids = np.floor((np.c_[pa.x, pa.y, pa.z] - g['xmin']) / g['cell_size'])
    groups = {}
    for i, key in enumerate(map(tuple, ids)):
        groups.setdefault(key, []).append(i)
    assert sorted(groups.values()) == [[0, 6], [1, 8], [2], [3, 7, 9], [4, 5]]


def test_nnps_corner_cases():
    # test_nnps.py:1250-1391
    pa = get_particle_array_wcsph(name='a', x=np.array([0.131, 0.359]),
                                  y=np.array([1.544, 1.809]),
                                  z=np.array([-3.6489999, -2.8559999]),
                                  h=np.ones(2))
    o = orc.Oracle([pa], 3, radius_scale=0.7)
    o.update_domain()
    o.nnps_update()
    for i in range(2):
        assert np.array_equal(np.sort(o.neighbors(0, 0, i)),
                              np.sort(o.brute_neighbors(0, 0, i)))
    # many particles in one cell: every particle neighbours every other
    rs = np.random.RandomState(1)
    n = 2 ** 11
    pb = get_particle_array_wcsph(name='b', x=rs.uniform(0, 0.1, n),
                                  y=rs.uniform(0, 0.1, n),
                                  z=rs.uniform(0, 0.1, n), h=np.ones(n))
    o = orc.Oracle([pb], 3, 'CubicSpline')
    o.update_domain()
    o.nnps_update()
    assert len(o.neighbors(0, 0, 5)) == n
    # too many cells -> error (linked_list_nnps.pyx:336-343, test_nnps.py:1019-1026)
    pc = get_particle_array_wcsph(name='c', x=np.array([0.0, 1e6]),
                                  y=np.array([0.0, 1e6]), z=np.array([0.0, 1e6]),
                                  h=np.full(2, 0.5))
    o = orc.Oracle([pc], 3, 'CubicSpline')
    o.update_domain()
    with pytest.raises(RuntimeError):
        o.nnps_update()


def test_dt_rules():
    # pysph/sph/tests/test_integrator.py:184-200: dt = cfl * h / max(dt_cfl)
    pa = get_particle_array_wcsph(name='f', x=np.zeros(4), h=np.full(4, 0.1))
    pa.dt_cfl[:] = [1.0, 2.0, 4.0, 3.0]
    s = orc.WCSPHOracleSolver([pa], dict(fluids=['f'], solids=[], dim=1, dt0=1.0,
                                         cfl=0.3, rho0=1.0, c0=1.0, gamma=7.0))
    assert abs(s._compute_timestep() - 0.3 * 0.1 / 4.0) < 1e-16
    pa.dt_force[:] = 1e6   # sqrt(h / sqrt(f)) = sqrt(0.1/1000) = 0.01 < 0.025
    assert abs(s._compute_timestep() - 0.3 * math.sqrt(0.1 / 1000.0)) < 1e-16


# ---------------------------------------------------------------------------
# EDAC scheme, transport-velocity branch (SURVEY.md 8f-1): the oracle against the
# reference's EDACScheme.get_equations() + equation bodies (oracle/gen_golden.py)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('idx', range(4))
def test_edac_evaluation_matches_reference_bodies(idx):
    from helpers import EDAC_FIELDS, edac_arrays_from_dict
    case = load_golden('edac_cases.json')[idx]
    p = case['params']
    # the equations the reference scheme emitted are the ones the oracle driver assumes
    want = ['MomentumEquationPressureGradient']
    if p['alpha'] > 0:
        want.append('MomentumEquationArtificialViscosity')
    if p['nu'] > 0:
        want.append('MomentumEquationViscosity')
    want += ['MomentumEquationArtificialStress', 'EDACEquation']
    assert p['groups'][1] == want * len(p['fluids'])
    assert p['groups'][0] == (['SummationDensity'] + (['ComputeAveragePressure'] if p['bql'] else [])) * len(p['fluids'])
    assert p['group_real'] == [False, True]
    pas = edac_arrays_from_dict(case['inputs'])
    s = orc.EDACOracleSolver(pas, dict(p, dt=1e-3), case['kernel'])
    s.t = p['t']
    s.evaluate()
    for pa in pas:
        ref = case['outputs'][pa.name]
        for f in EDAC_FIELDS:
            got, wantv = pa.properties[f], np.array(ref[f])
            scale = max(np.max(np.abs(wantv)), 1e-300)
            assert np.max(np.abs(got - wantv)) <= 5e-12 * scale, (pa.name, f)


@pytest.mark.parametrize('idx', range(4))
def test_edac_solid_wall_evaluation_matches_reference_bodies(idx):
    """EDACScheme(fluids, solids=['wall']): the reference's own scheme method and the bodies of
    SourceNumberDensity, VolumeSummation, SolidWallPressureBC, SetWallVelocity,
    SolidWallNoSlipBC (+ the fluid equations with a wall among their sources)."""
    from helpers import EDAC_FIELDS, EDAC_WALL_FIELDS, edac_wall_arrays_from_dict
    case = load_golden('edac_wall_cases.json')[idx]
    p = case['params']
    # the Groups, equations and sources the reference emitted are what the oracle driver assumes
    g1 = ['SummationDensity', 'SourceNumberDensity', 'VolumeSummation', 'SolidWallPressureBC',
          'SetWallVelocity']
    g2 = ['MomentumEquationPressureGradient']
    s2 = [['fluid', 'wall']]
    if p['alpha'] > 0:
        g2.append('MomentumEquationArtificialViscosity'); s2.append(['fluid', 'wall'])
    if p['nu'] > 0:
        g2 += ['MomentumEquationViscosity', 'SolidWallNoSlipBC']; s2 += [['fluid'], ['wall']]
    g2 += ['MomentumEquationArtificialStress', 'EDACEquation']; s2 += [['fluid'], ['fluid', 'wall']]
    want = [g1] + ([['ComputeAveragePressure']] if p['bql'] else []) + [g2]
    assert p['groups'] == want
    assert p['group_real'] == [False] + ([True] if p['bql'] else []) + [True]
    assert p['sources'][0] == [['fluid', 'wall'], ['fluid'], ['fluid', 'wall'], ['fluid'], ['fluid']]
    assert p['sources'][-1] == s2
    pas = edac_wall_arrays_from_dict(case['inputs'])
    s = orc.EDACOracleSolver(pas, dict(p, dt=1e-3), case['kernel'])
    s.t = p['t']
    s.evaluate()
    for pa, fields in zip(pas, (EDAC_FIELDS, EDAC_WALL_FIELDS)):
        ref = case['outputs'][pa.name]
        for f in fields:
            got, wantv = pa.properties[f], np.array(ref[f])
            scale = max(np.max(np.abs(wantv)), 1e-300)
            assert np.max(np.abs(got - wantv)) <= 5e-12 * scale, (pa.name, f)


@pytest.mark.parametrize('idx', range(4))
def test_edac_external_flow_evaluation_matches_reference_bodies(idx):
    """EDACScheme(..., pb=0): the external-flow branch (wc/edac.py:882-971) -- number-density
    MomentumEquation, EDACEquation, XSPHCorrection(sources=[the fluid itself]), walls,
    ClampWallPressure -- through the reference's own scheme method and bodies."""
    from helpers import EDAC_EXT_FIELDS, EDAC_WALL_FIELDS, edac_ext_arrays_from_dict
    case = load_golden('edac_ext_cases.json')[idx]
    p = case['params']
    fl, walls = p['fluids'], p['solids']
    g1 = ['SummationDensity'] * len(fl)
    for w in walls:
        g1 += ['SourceNumberDensity', 'VolumeSummation', 'SolidWallPressureBC', 'SetWallVelocity']
        if p['clamp_p']:
            g1.append('ClampWallPressure')
    per_fluid = ['MomentumEquation']
    if p['alpha'] > 0:
        per_fluid.append('MomentumEquationArtificialViscosity')
    if p['nu'] > 0:
        per_fluid.append('MomentumEquationViscosity')
        if walls:
            per_fluid.append('SolidWallNoSlipBC')
    per_fluid += ['EDACEquation', 'XSPHCorrection']
    assert p['groups'] == [g1, per_fluid * len(fl)] and p['group_real'] == [False, True]
    # XSPH takes the fluid itself as its only source
    assert [s_ for s_, n in zip(p['sources'][1], p['groups'][1]) if n == 'XSPHCorrection'] == [[f] for f in fl]
    pas = edac_ext_arrays_from_dict(case['inputs'])
    s = orc.EDACOracleSolver(pas, dict(p, dt=1e-3), case['kernel'])
    s.t = p['t']
    s.evaluate()
    for pa in pas:
        ref = case['outputs'][pa.name]
        for f in (EDAC_WALL_FIELDS if pa.name in walls else EDAC_EXT_FIELDS):
            got, wantv = pa.properties[f], np.array(ref[f])
            scale = max(np.max(np.abs(wantv)), 1e-300)
            assert np.max(np.abs(got - wantv)) <= 5e-12 * scale, (pa.name, f)


def test_edac_step_matches_reference_bodies():
    from pysph_b200.particle_array import get_particle_array_edac_ext
    g = load_golden('edac_ext_stepper.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        a = g[key]
        pa = get_particle_array_edac_ext(name='f', **dict((k, np.array(v)) for k, v in a['inputs'].items()))
        o = orc.Oracle([pa], 3, 'CubicSpline')
        o.stage_edac(0, which, g['dt'])
        for k, v in a['outputs'].items():
            assert np.max(np.abs(pa.properties[k] - np.array(v))) <= 1e-15 * max(1.0, np.max(np.abs(v))), (key, k)


def test_edac_tvf_step_matches_reference_bodies():
    from pysph_b200.particle_array import get_particle_array_edac
    g = load_golden('edac_stepper.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        pa = get_particle_array_edac(name='f', **props)
        o = orc.Oracle([pa], 3)
        o.stage_tvf(0, which, g['dt'])
        for k, v in g['outputs'][key].items():
            assert np.allclose(pa.properties[k], v, rtol=1e-15, atol=0), (key, k)


# ---------------------------------------------------------------------------
# elastic dynamics (SURVEY.md 8f-2): the restatement of
# ElasticSolidsScheme's loops against the reference's scheme method + bodies, with the
# reference's own compiled linalg3 eigen solver behind MonaghanArtificialStress
# ---------------------------------------------------------------------------
SOLID_FIELDS = ['p', 'arho', 'au', 'av', 'aw', 'ax', 'ay', 'az'] + \
    ['v%d%d' % (i, j) for i in range(3) for j in range(3)] + \
    [pre + k for pre in ('r', 'as') for k in ('00', '01', '02', '11', '12', '22')]


def _solid_arrays(case):
    from pysph_b200.particle_array import get_particle_array_elastic_dynamics
    pas = []
    for name in case['params']['names']:
        a = case['inputs'][name]
        props = dict((k, np.array(v, dtype=float)) for k, v in a.items() if k[0] != '_')
        consts = dict((k, v[0]) for k, v in case['params']['constants'][name].items())
        pa = get_particle_array_elastic_dynamics(name=name, constants=consts, **props)
        pa.set_num_real_particles(a['_n_real'])
        pas.append(pa)
    return pas


@pytest.mark.parametrize('idx', range(6))
def test_elastic_dynamics_matches_reference_bodies(idx):
    case = load_golden('solid_cases.json')[idx]
    p = case['params']
    assert p['groups'][0][:3] == ['IsothermalEOS', 'VelocityGradient3D' if p.get('grad3d')
                                  else 'VelocityGradient2D', 'MonaghanArtificialStress']
    assert p['groups'][1][:5] == ['ContinuityEquation', 'MomentumEquationWithStress',
                                  'MonaghanArtificialViscosity',
                                  'HookesDeviatoricStressRate', 'XSPHCorrection']
    assert p['group_real'] == [True, True]
    pas = _solid_arrays(case)
    o = orc.Oracle(pas, p['dim'], case['kernel'])
    o.update_domain()
    o.nnps_update()
    idxs = list(range(len(pas)))                 # sources: rigid solids + elastic solids
    elastic = [i for i, pa in enumerate(pas) if pa.name in p['elastic']]
    P = o.solid_program(elastic, idxs, eps=p['eps'], alpha=p['alpha'], beta=p['beta'],
                        eps_xsph=p['eps_xsph'], grad3d=p.get('grad3d', False))
    o.solid_group1(P)
    o.solid_group2(P)
    for pa in pas:
        ref = case['outputs'][pa.name]
        nr = ref['_n_real']
        for f in SOLID_FIELDS:
            want = np.array(ref[f])[:nr]
            got = pa.properties[f][:nr]
            if pa.name in p['solids']:           # a rigid solid is a destination of nothing
                assert np.array_equal(got, want) and \
                    np.array_equal(want, np.array(case['inputs'][pa.name][f])[:nr]), (pa.name, f)
                continue
            scale = max(np.max(np.abs(want)), 1e-300)
            assert np.max(np.abs(got - want)) <= 1e-10 * scale, (pa.name, f)
        # destinations are the real particles only: ghosts untouched
        assert np.all(pa.properties['au'][nr:] == 0.0)


def test_solid_mech_step_matches_reference_bodies():
    from pysph_b200.particle_array import get_particle_array_elastic_dynamics
    g = load_golden('solid_stepper.json')
    for which, key in ((0, 'initialize'), (1, 'stage1'), (2, 'stage2')):
        props = dict((k, np.array(v)) for k, v in g['inputs'].items())
        pa = get_particle_array_elastic_dynamics(name='f', **props)
        o = orc.Oracle([pa], 3)
        o.stage_solid(0, which, g['dt'])
        for k, v in g['outputs'][key].items():
            assert np.allclose(pa.properties[k], v, rtol=1e-15, atol=0), (key, k)


def test_eigen_sym3_against_numpy():
    rs = np.random.RandomState(4)
    for t in range(50):
        a = rs.normal(size=(3, 3)) * 10.0 ** rs.randint(-6, 6)
        a = a + a.T
        if t % 10 == 0:
            a = np.diag([2.0, 2.0, -1.0]) * a[0, 0]          # repeated eigenvalue
        d, v = orc.eigen_sym3(a)
        s = max(np.max(np.abs(a)), 1e-300)
        assert np.max(np.abs(v @ np.diag(d) @ v.T - a)) <= 1e-13 * s
        assert np.max(np.abs(v.T @ v - np.eye(3))) <= 1e-14
        assert np.max(np.abs(np.sort(d) - np.linalg.eigvalsh(a))) <= 1e-13 * s


# ---------------------------------------------------------------------------
# stand-alone MonaghanArtificialViscosity (basic_equations.py:195-257): the ORC_EQ_AV
# branch, which the WCSPH scheme never takes (its MomentumEquation carries the AV)
# ---------------------------------------------------------------------------
def run_oracle_monaghan_case(case):
    p = case['params']
    pas = arrays_from_dict(case['inputs'], order=tuple(p['names']))
    o = orc.Oracle(pas, case['dim'], case['kernel'])
    o.update_domain()
    o.nnps_update()
    for a in range(len(pas)):
        o.eos(a, 0, p['rho0'], p['c0'], p['gamma'], 0.0, real_only=False)
    pairs = o.pair_pass([(orc.EQ_CONT, 0, [0, 1]), (orc.EQ_AV, 0, [0, 1]),
                         (orc.EQ_XSPH, 0, [0])], real_only=True, alpha=p['alpha'],
                        beta=p['beta'], eps_xsph=p['eps_xsph'])
    return pas, pairs


@pytest.mark.parametrize('idx', range(2))
def test_monaghan_av_matches_reference_bodies(idx):
    case = load_golden('monaghan_av_cases.json')[idx]
    pas, pairs = run_oracle_monaghan_case(case)
    assert pairs > 0
    ref = case['outputs']['fluid']
    for f in ('arho', 'au', 'av', 'aw', 'ax', 'ay', 'az', 'p', 'cs'):
        got, want = pas[0].properties[f], np.array(ref[f])
        scale = max(np.max(np.abs(want)), 1e-300)
        assert np.max(np.abs(got - want)) <= 2e-12 * scale, f
    assert np.max(np.abs(ref['au'])) > 1.0       # the AV term is active in the fixture
