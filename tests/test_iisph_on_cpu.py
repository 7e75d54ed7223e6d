"""IISPHScheme without a GPU: the fp64 oracle against the fixture the reference's own bodies made,
the fixture's coverage and its generator, the program translation, and the checks of
tests/test_gpu_iisph.py on the library emulation (the loader of test_library_on_cpu.py),
smaller."""
import json
import os

import numpy as np
import pytest

import iisph_oracle as orc
import test_gpu_iisph as t
from helpers import load_golden
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

REF = os.environ.get('PYSPH_REFERENCE', '/root/reference')


# ---- the oracle against the reference ------------------------------------------------------------
def _oracle_case(c):
    arrays = {}
    for name, a in c['inputs'].items():
        A = dict((k, np.array(v, dtype=float)) for k, v in a.items())
        for k in ('V', 'p'):
            A.setdefault(k, np.zeros(len(A['x'])))
        arrays[name] = A
    L = [c['L'] if d < c['dim'] else 0.0 for d in range(3)]
    it, hist = orc.evaluate(arrays, c['fluids'], c['solids'], c['rho0'], c['kernel'], c['dim'],
                            c['dt'], nu=c['nu'], g=c['g'], omega=c['omega'],
                            tolerance=c['tolerance'], L=L)
    for f in c['fluids']:
        orc.stage(arrays[f], c['dt'])
    return arrays, it, hist


def test_oracle_matches_the_reference_fixture():
    """tests/iisph_oracle.py against the reference's bodies to 1e-12 of each field's largest
    magnitude, the iteration count and the compression of every iteration"""
    for c in load_golden('iisph_cases.json'):
        arrays, it, hist = _oracle_case(c)
        assert it == c['iterations'], (c['kernel'], c['dim'])
        for got, want in zip(hist, c['compression']):
            for f in c['fluids']:
                assert abs(got[f] - want[f]) <= 1e-12 * max(want[f], 1e-300), (c['kernel'], c['dim'])
        for name, out in c['outputs'].items():
            for k, v in out.items():
                want = np.array(v)
                got = arrays[name][k[5:] if k.startswith('step_') else k]
                scale = max(float(np.max(np.abs(want))), 1e-300)
                assert float(np.max(np.abs(got - want))) <= 1e-12 * scale, (c['kernel'], c['dim'], name, k)


def test_fixture_covers_the_cases():
    """every kernel in 2-D and 3-D; a fluid block alone, fluid over a wall with nu = 0 and
    nu > 0, a periodic box with has_ghosts, two fluid arrays; a case that stops at
    min_iterations and one that reaches max_iterations; h varies by +-10 %"""
    cases = load_golden('iisph_cases.json')
    assert {(c['kernel'], c['dim']) for c in cases} == {(k, d) for k in orc.KERNELS for d in (2, 3)}
    assert {c['kind'] for c in cases} == {'block', 'tank', 'periodic', 'two'}
    assert any(c['solids'] and c['nu'] == 0 for c in cases) and any(c['solids'] and c['nu'] > 0 for c in cases)
    assert any(c['iterations'] == 2 and c['tolerance'] >= 1.0 for c in cases)   # min_iterations
    assert any(c['iterations'] == 30 for c in cases)
    assert any(2 < c['iterations'] < 30 for c in cases)
    for c in cases:
        h = np.array(c['inputs']['fluid']['h'])
        assert h.max() / h.min() > 1.1


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, 'pysph', 'sph', 'iisph.py')),
                    reason='the reference is not present')
def test_generator_reproduces_the_fixture():
    """tests/gen_iisph_golden.py, run on the reference, writes what the fixture holds (the
    cheapest case of each geometry)"""
    import gen_iisph_golden as gen
    kernels, iisph = gen.load()
    import math
    iisph.sqrt, iisph.fabs = math.sqrt, math.fabs
    cases = load_golden('iisph_cases.json')
    for c in cases:
        if c['dim'] != 2 or c['kind'] == 'periodic':
            continue
        got = gen.run_case(kernels, iisph, c['kernel'], c['dim'], c['kind'], c['seed'], nu=c['nu'],
                           tolerance=c['tolerance'], g=tuple(c['g']), dt=c['dt'])
        assert json.loads(json.dumps(got)) == c


# ---- the translation -----------------------------------------------------------------------------
def test_translation_and_fallback():
    t.check_iisph_named_group_outside_the_scheme_is_generic()


def test_translation_of_every_variant():
    """nu > 0, no solids, has_ghosts, two fluids: one op each, with the Group's iteration
    limits; a changed parameter inside one Group is not the scheme"""
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    for kw in (dict(nu=0.1), dict(has_ghosts=True), dict(omega=0.7, tolerance=1e-4)):
        for fluids, solids in ((['f'], ['w']), (['f', 'g'], []), (['f', 'g'], ['w', 'v'])):
            eqs = pb.IISPHScheme(fluids, solids, 2, 1000.0, gy=-9.81, **kw).get_equations()
            eqs[-2].max_iterations = 12
            ops = build_program(eqs, ['f', 'g', 'w', 'v'], 2)
            assert [op[0] for op in ops] == ['iisph'], (kw, fluids, solids)
            prog = ops[0][1]
            assert prog.max_iterations == 12 and prog.nu == kw.get('nu', 0.0)
            # get_equations does not hand the scheme's omega to PressureSolve (iisph.py:597-599)
            assert prog.omega == 0.5 and prog.tolerance == kw.get('tolerance', 1e-2)
            assert prog.fluid_mask == sum(1 << ['f', 'g', 'w', 'v'].index(a) for a in fluids)
            assert prog.solid_mask == sum(1 << ['f', 'g', 'w', 'v'].index(a) for a in solids)
    # a parameter changed in one Group: not the scheme (each Group then goes its own way, and
    # the first, NumberDensity, has no kernel)
    eqs = pb.IISPHScheme(['f'], ['w'], 2, 1000.0).get_equations()
    eqs[4].equations[2].rho0 = 999.0             # ComputeRhoBoundary
    with pytest.raises(NotImplementedError, match='NumberDensity'):
        build_program(eqs, ['f', 'w'], 2)
    eqs = pb.IISPHScheme(['f'], ['w'], 2, 1000.0).get_equations()
    eqs[4].real = False
    with pytest.raises(NotImplementedError, match='NumberDensity'):
        build_program(eqs, ['f', 'w'], 2)


def test_integrators_and_steppers():
    import pysph_b200 as pb
    integ = pb.EulerIntegrator(fluid=pb.IISPHStep())
    assert integ.steppers_supported[-1] == 'IISPHStep'
    with pytest.raises(NotImplementedError):
        pb.PECIntegrator(fluid=pb.IISPHStep())
    with pytest.raises(NotImplementedError, match='EulerStep'):
        pb.EulerIntegrator(fluid=pb.WCSPHStep()).stage1()
    pa = pb.get_particle_array_iisph(name='f', x=[0.0, 1.0])
    assert 'tmp_comp' in pa.constants and 'piter' in pa.properties and 'dt_force' in pa.properties
    assert pa.output_property_arrays == ['x', 'y', 'z', 'u', 'v', 'w', 'rho', 'h', 'm', 'p', 'pid',
                                        'au', 'av', 'aw', 'tag', 'gid', 'V']


# ---- the GPU checks on the library emulation -----------------------------------------------------
def test_fixture_on_the_emulation(emulated_library):
    for c in load_golden('iisph_cases.json'):
        t.check_fixture(c)


@pytest.mark.parametrize('kernel', orc.KERNELS)
def test_one_evaluation_on_the_emulation(emulated_library, kernel):
    for case in (t.dam2d(0.25), t.dam3d(0.25)):
        case['kernel'] = kernel
        t.check_one_evaluation(case, tolerance=1e-3)


SMALL = {
    'dam2d': (lambda: t.dam2d(0.1), dict(tolerance=1e-3), 20),
    'dam3d': (lambda: t.dam3d(0.2), dict(tolerance=1e-3), 8),
    'tg2': (lambda: t.taylor_green(12, 2), {}, 10),
    'tg3': (lambda: t.taylor_green(8, 3), {}, 4),
    'max': (lambda: t.dam2d(0.1), dict(tolerance=1e-9), 3),
}


@pytest.mark.parametrize('name', sorted(SMALL))
def test_runs_against_the_oracle_on_the_emulation(emulated_library, name):
    t.check_run(name, SMALL)


def test_host_dt_is_device_dt_on_the_emulation(emulated_library):
    t.check_host_dt_is_device_dt(t.dam2d(0.15), 5)


def test_two_runs_bitwise_on_the_emulation(emulated_library):
    t.check_two_runs_bitwise(t.dam2d(0.15), 5)


def test_repeat_starts_from_the_steps_pressure_on_the_emulation(emulated_library):
    t.check_repeat_starts_from_the_steps_pressure(t.dam2d(0.12))


def test_dump_and_restart_on_the_emulation(emulated_library, tmp_path):
    case = t.dam2d(0.12)
    case['adaptive'] = False
    t.check_dump_and_restart(case, 3, tmp_path)


def test_refusals_on_the_emulation(emulated_library):
    t.check_refusals(t.dam2d(0.25))
    t.check_ghosts_and_1d_refused()


def test_property_ids_on_the_emulation(emulated_library):
    t.check_property_ids()
