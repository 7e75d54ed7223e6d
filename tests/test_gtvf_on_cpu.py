"""GTVFScheme without a GPU: the fp64 oracle against the fixture the reference's own bodies made,
the fixture's coverage and its generator, the translation of the reference's own objects, and the
checks of tests/test_gpu_gtvf.py on the library emulation (the loader of
test_library_on_cpu.py), smaller."""
import json
import os

import numpy as np
import pytest

import gtvf_oracle as orc
import test_gpu_gtvf as t
from helpers import load_golden
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

REF = os.environ.get('PYSPH_REFERENCE', '/root/reference')
HAVE_REF = os.path.exists(os.path.join(REF, 'pysph', 'sph', 'wc', 'gtvf.py'))


def _arrays(c):
    arrays = {}
    for name, a in c['inputs'].items():
        A = dict((k, np.array(v, dtype=float)) for k, v in a.items())
        n = len(A['x'])
        for k in ('z', 'u', 'v', 'w', 'uhat', 'vhat', 'what', 'au', 'av', 'aw', 'auhat', 'avhat',
                  'awhat', 'p', 'rho0'):
            A.setdefault(k, np.zeros(n))
        arrays[name] = A
    return arrays


def _close(got, want, tag, rel):
    want = np.array(want, dtype=float)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin), tag
    if not fin.any():
        return
    scale = max(float(np.max(np.abs(want[fin]))), 1e-300)
    assert float(np.max(np.abs(got[fin] - want[fin]))) <= rel * scale, tag


def test_oracle_matches_the_reference_fixture():
    """tests/gtvf_oracle.py against the reference's bodies to 1e-12 of each field's largest
    magnitude: both evaluations, and the 5 integrator steps of the 2-D wall cases"""
    for c in load_golden('gtvf_cases.json'):
        L = [c['L'] if d < c['dim'] else 0.0 for d in range(3)]
        kw = dict(c0=c['c0'], alpha=c['alpha'], nu=c['nu'], g=c['g'], L=L)
        arrays = _arrays(c)
        orc.evaluate0(arrays, c['fluids'], c['solids'], c['kernel'], c['dim'], L=L)
        for name, out in c['eval0'].items():
            for k, v in out.items():
                _close(arrays[name][k], v, (c['kernel'], c['dim'], 0, name, k), 1e-12)
        orc.evaluate1(arrays, c['fluids'], c['solids'], c['kernel'], c['dim'], c['rho0'], c['pref'], **kw)
        for name, out in c['eval1'].items():
            for k, v in out.items():
                rel = 1e-12 if k != 'rho' else 1e-12 * 1e3     # (rho ~ 1e3, its change ~ 1e2)
                _close(arrays[name][k], v, (c['kernel'], c['dim'], 1, name, k), rel)
        if c['steps']:
            s = orc.Solver(_arrays(c), c['fluids'], c['solids'], c['kernel'], c['dim'], c['dt'],
                           c['rho0'], c['pref'], **kw)
            s.initialise()
            for _ in range(c['steps']):
                s.step()
            for name, out in c['stepped'].items():
                for k, v in out.items():
                    _close(s.arrays[name][k], v, (c['kernel'], c['dim'], 'steps', name, k), 1e-10)


def test_fixture_covers_the_cases():
    """every kernel in 2-D and 3-D; a block, a fluid over a 4-layer wall with wall rho0 = 0 and
    with rho0 = rho, alpha > 0 beside walls, a periodic box with nu > 0; both branches of
    min(10 |p|, pref); h varies by +-10 %; integrator steps"""
    cases = load_golden('gtvf_cases.json')
    assert {(c['kernel'], c['dim']) for c in cases} == {(k, d) for k in orc.KERNELS for d in (2, 3)}
    assert {c['kind'] for c in cases} == {'block', 'tank', 'tank_rho', 'periodic'}
    assert any(c['kind'] == 'tank' and c['alpha'] > 0 for c in cases)
    assert any(c['kind'] == 'periodic' and c['nu'] > 0 for c in cases)
    assert any(c['steps'] for c in cases)
    both = 0
    for c in cases:
        p = np.array(c['eval1']['fluid']['p'])
        both += bool(np.any(10 * np.abs(p) < c['pref']) and np.any(10 * np.abs(p) > c['pref']))
        h = np.array(c['inputs']['fluid']['h'])
        assert h.max() / h.min() > 1.1
        if c['kind'] == 'tank':
            assert not np.all(np.isfinite(c['eval1']['fluid']['rhodiv']))   # wall rho0 = 0
    assert both >= 6


@pytest.mark.skipif(not HAVE_REF, reason='the reference is not present')
def test_generator_reproduces_the_fixture():
    """tests/gen_gtvf_golden.py, run on the reference, writes what the fixture holds (the 2-D
    cases without steps)"""
    import gen_gtvf_golden as gen
    kernels, gtvf = gen.load()
    for c in load_golden('gtvf_cases.json'):
        if c['dim'] != 2 or c['steps']:
            continue
        got = gen.run_case(kernels, gtvf, c['kernel'], c['dim'], c['kind'], c['seed'], c['pref'],
                           alpha=c['alpha'], nu=c['nu'], g=tuple(c['g']), dt=c['dt'])
        assert json.loads(json.dumps(got)) == c


@pytest.mark.skipif(not HAVE_REF, reason='the reference is not present')
def test_translation_of_the_reference_objects():
    """the reference's own GTVFScheme.get_equations(): each evaluation is one op, with the same
    program as this package's scheme gives"""
    import gen_gtvf_golden as gen
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    _, gtvf = gen.load()
    for solids, alpha, nu in ((['w'], 0.1, 0.0), ([], 0.0, 0.05), (['w'], 0.0, 0.0)):
        ref = gtvf.GTVFScheme(['f'], solids, 2, 1000.0, 10.0, nu, None, 1e5, gy=-9.81, alpha=alpha)
        ours = pb.GTVFScheme(['f'], solids, 2, 1000.0, 10.0, nu, None, 1e5, gy=-9.81, alpha=alpha)
        for k in (0, 1):
            a = build_program(ref.get_equations().groups[k], ['f', 'w'], 2)
            b = build_program(ours.get_equations().groups[k], ['f', 'w'], 2)
            assert [(op[0], op[2]) for op in a] == [('gtvf', k)]
            assert bytes(a[0][1]) == bytes(b[0][1])


def test_translation_and_integrators():
    t.check_translation()
    import pysph_b200 as pb
    assert pb.GTVFIntegrator.steppers_supported == ('GTVFStep',)
    for cls in (pb.PECIntegrator, pb.EPECIntegrator, pb.TVDRK3Integrator, pb.EulerIntegrator):
        assert 'GTVFStep' not in cls.steppers_supported
    pa = pb.get_particle_array_gtvf(name='f', x=[0.0, 1.0])
    assert pa.sigma.size == 18 and 'rhodiv' in pa.properties
    assert pa.output_property_arrays == ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'p', 'h', 'm', 'au',
                                         'av', 'aw', 'pid', 'gid', 'tag']


# ---- the GPU checks on the library emulation -----------------------------------------------------
def test_fixture_on_the_emulation(emulated_library):
    for c in load_golden('gtvf_cases.json'):
        t.check_fixture(c)


SMALL = {
    'dam2d': (lambda: t.dam2d(0.2), 10),
    'dam3d': (lambda: t.dam3d(0.25), 4),
    'tg2': (lambda: t.taylor_green(12, 2), 10),
    'tg3': (lambda: t.taylor_green(6, 3), 3),
}


@pytest.mark.parametrize('name', sorted(SMALL))
def test_runs_against_the_oracle_on_the_emulation(emulated_library, name):
    t.check_run(name, SMALL)


def test_first_step_on_the_emulation(emulated_library):
    t.check_first_step(t.dam2d(0.2))


def test_host_dt_is_device_dt_on_the_emulation(emulated_library):
    t.check_host_dt_is_device_dt(t.dam2d(0.25), 4)


def test_two_runs_bitwise_on_the_emulation(emulated_library):
    t.check_two_runs_bitwise(t.dam2d(0.25), 4)


def test_repeat_keeps_the_stage_density_on_the_emulation(emulated_library):
    t.check_repeat_keeps_the_stage_density(t.dam2d(0.2))


def test_dump_and_restart_on_the_emulation(emulated_library, tmp_path):
    t.check_dump_and_restart(t.dam2d(0.25), 2, tmp_path)


def test_refusals_on_the_emulation(emulated_library):
    t.check_refusals(t.dam2d(0.25))
    t.check_ghosts_and_1d_refused()


def test_property_ids_on_the_emulation(emulated_library):
    t.check_property_ids()
