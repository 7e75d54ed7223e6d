"""CRKSPHScheme without a GPU: the fp64 oracle against the fixture the reference's own bodies made,
the reproducing property and momentum conservation on the oracle, the fixture's coverage and its
generator, the translation of the reference's own objects, and the checks of
tests/test_gpu_crksph.py on the library emulation (the loader of test_library_on_cpu.py),
smaller."""
import json
import os

import numpy as np
import pytest

import crksph_oracle as orc
import test_gpu_crksph as t
from helpers import load_golden
from test_library_on_cpu import emulated_library  # noqa: F401  (the fixture)

REF = os.environ.get('PYSPH_REFERENCE', '/root/reference')
HAVE_REF = os.path.exists(os.path.join(REF, 'pysph', 'sph', 'wc', 'crksph.py'))


def _arrays(c):
    A = dict((k, np.array(v, dtype=float)) for k, v in c['inputs']['fluid'].items())
    n = len(A['x'])
    for k in ('z', 'u', 'v', 'w', 'u0', 'v0', 'w0', 'e'):
        A.setdefault(k, np.zeros(n))
    return A


def _flat(A, k, d):
    if k in ('bi', 'gradai'):
        return A[k][:, :d].ravel()
    if k in ('gradbi', 'gradv'):
        return A[k][:, :d, :d].ravel()
    return A[k]


def _close(got, want, tag, rel):
    want = np.array(want, dtype=float)
    scale = float(np.max(np.abs(want)))
    if scale == 0.0:
        assert np.array_equal(got, want), tag
        return
    assert float(np.max(np.abs(got - want))) <= rel * scale, tag


def _L(c):
    return [c['L'] if q < c['dim'] else 0.0 for q in range(3)]


def test_oracle_matches_the_reference_fixture():
    """tests/crksph_oracle.py against the reference's bodies to 1e-12 of each field's largest
    magnitude: both evaluations, and the integrator steps"""
    for c in load_golden('crksph_cases.json'):
        d, L = c['dim'], _L(c)
        A = _arrays(c)
        orc.evaluate0(A, c['kernel'], d, gamma=c['gamma'], g=c['g'], nu=c['nu'], L=L)
        for k, v in c['eval0']['fluid'].items():
            _close(_flat(A, k, d), v, (c['kernel'], d, c['kind'], 0, k), 1e-12)
        orc.evaluate1(A, c['kernel'], d, gamma=c['gamma'], L=L)
        _close(A['ae'], c['eval1']['fluid']['ae'], (c['kernel'], d, c['kind'], 1), 1e-12)
        if c['steps']:
            s = orc.Solver(_arrays(c), c['kernel'], d, c['dt'], L=L, gamma=c['gamma'], g=c['g'],
                           nu=c['nu'])
            s.initialise()
            for _ in range(c['steps']):
                s.step()
            for k, v in c['stepped']['fluid'].items():
                _close(s.A[k], v, (c['kernel'], d, 'steps', k), 1e-12)


def test_fixture_covers_the_cases():
    """every kernel in 2-D and 3-D; a block, a fluid at rest (the limiter's 0 / 0), a periodic
    box in 2-D and 3-D; e = 0 and e > 0; nu > 0; gravity; h varying by +-10 %; integrator steps"""
    cases = load_golden('crksph_cases.json')
    assert {(c['kernel'], c['dim']) for c in cases} == {(k, d) for k in orc.KERNELS for d in (2, 3)}
    assert {(c['kind'], c['dim']) for c in cases} >= {('periodic', 2), ('periodic', 3),
                                                      ('rest', 2), ('block', 2), ('block', 3)}
    assert {c['e0'] > 0 for c in cases} == {True, False}
    assert any(c['nu'] > 0 for c in cases) and any(any(c['g']) for c in cases)
    assert any(c['steps'] for c in cases)
    for c in cases:
        h = np.array(c['inputs']['fluid']['h'])
        assert h.max() / h.min() > 1.1
        gv = np.array(c['eval0']['fluid']['gradv'])
        assert np.all(gv == 0.0) == (c['kind'] == 'rest')
        p = np.array(c['eval0']['fluid']['p'])
        assert np.all(p == 0.0) == (c['e0'] == 0.0)


def test_reproducing_property_on_the_oracle():
    """pysph/sph/tests/test_kernel_corrections.py::test_crksph: for interior particles of a
    perturbed lattice, after the pre-step, sum_j V_j W^R_ij = 1 and sum_j V_j x_ij W^R_ij = 0 to
    1e-12"""
    for dim, kernel in ((2, 'CubicSpline'), (2, 'QuinticSpline'), (3, 'WendlandQuintic')):
        case = t.block(0.05 if dim == 2 else 0.1, dim)
        case['kernel'] = kernel
        o = t.oracle_of(case)
        o.initialise()
        A = o.A
        i, j, x, r, hij = orc.pairs(A, A, kernel)
        w, _ = orc._wd(kernel, dim, x, r, hij)
        wr = A['ai'][i] * (1 + np.einsum('pa,pa->p', A['bi'][i], x)) * w / A['V'][j]
        n = len(A['x'])
        s0, s1 = orc._sum(i, n, wr), orc._sum(i, n, wr[:, None] * x)
        inner = np.ones(n, dtype=bool)
        margin = orc.RADIUS[kernel] * 1.1 * np.max(A['h'])
        for c in 'xyz'[:dim]:
            inner &= (A[c] > A[c].min() + margin) & (A[c] < A[c].max() - margin)
        assert inner.sum() > 0
        assert np.max(np.abs(s0[inner] - 1.0)) < 1e-12
        assert np.max(np.abs(s1[inner])) < 1e-12 * case['dx']


def test_momentum_conservation_on_the_oracle():
    """uniform h in a periodic box without gravity: sum_i m_i a_i = 0 to round-off.  With h
    varying it does not hold: MomentumEquation divides both mu_i and mu_j by |x_ij|^2 / h_i, so
    Q_j of the pair (i, j) is not Q_i of (j, i)"""
    for e0 in (0.0, 1.0):
        case = t.taylor_green(12, 2, perturb=0.1, e0=e0)
        o = t.oracle_of(case)
        o.initialise()
        A = o.A
        scale = float(np.sum(A['m'] * np.hypot(A['au'], A['av'])))
        for k in ('au', 'av'):
            assert abs(float(np.sum(A['m'] * A[k]))) <= 1e-13 * scale
    case = t.taylor_green(12, 2, perturb=0.1, e0=1.0)
    case['arrays'][0].h[:] *= 1.0 + 0.1 * np.random.RandomState(1).uniform(-1, 1, case['arrays'][0].h.size)
    o = t.oracle_of(case)
    o.initialise()
    A = o.A
    scale = float(np.sum(A['m'] * np.hypot(A['au'], A['av'])))
    assert abs(float(np.sum(A['m'] * A['au']))) > 1e-8 * scale


@pytest.mark.skipif(not HAVE_REF, reason='the reference is not present')
def test_generator_reproduces_the_fixture():
    """tests/gen_crksph_golden.py, run on the reference, writes what the fixture holds (the 2-D
    cases that are not periodic)"""
    import gen_crksph_golden as gen
    kernels, crksph = gen.load()
    for c in load_golden('crksph_cases.json'):
        if c['dim'] != 2 or c['L']:
            continue
        got = gen.run_case(kernels, crksph, c['kernel'], c['dim'], c['kind'], c['seed'],
                           e0=c['e0'], nu=c['nu'], g=tuple(c['g']), dt=c['dt'], steps=c['steps'])
        assert json.loads(json.dumps(got)) == c


@pytest.mark.skipif(not HAVE_REF, reason='the reference is not present')
def test_translation_of_the_reference_objects():
    """the reference's own CRKSPHScheme.get_equations(): each evaluation is one op, with the same
    program as this package's scheme gives"""
    import gen_crksph_golden as gen
    import pysph_b200 as pb
    from pysph_b200.program import build_program
    _, crksph = gen.load()
    for nu, ghosts in ((0.0, False), (0.05, True)):
        kw = dict(fluids=['f'], dim=2, nu=nu, rho0=1.0, h0=0.1, c0=10.0, p0=0.0, gy=-9.81,
                  has_ghosts=ghosts)
        ref, ours = crksph.CRKSPHScheme(**kw), pb.CRKSPHScheme(**kw)
        for k in (0, 1):
            a = build_program(ref.get_equations().groups[k], ['f'], 2)
            b = build_program(ours.get_equations().groups[k], ['f'], 2)
            assert [(op[0], op[2]) for op in a] == [('crksph', k)]
            assert bytes(a[0][1]) == bytes(b[0][1])


def test_translation_and_integrators():
    t.check_translation()


# ---- the GPU checks on the library emulation -----------------------------------------------------
def test_fixture_on_the_emulation(emulated_library):
    for c in load_golden('crksph_cases.json'):
        t.check_fixture(c)


SMALL = {
    'tg2': (lambda: t.taylor_green(10, 2), 4),
    'tg3': (lambda: t.taylor_green(5, 3, e0=1.0), 2),
    'block2': (lambda: t.block(0.2, 2), 4),
}


@pytest.mark.parametrize('name', sorted(SMALL))
def test_runs_against_the_oracle_on_the_emulation(emulated_library, name):
    t.check_run(name, SMALL)


def test_first_step_on_the_emulation(emulated_library):
    t.check_first_step(t.block(0.2, 2))


def test_host_dt_is_device_dt_on_the_emulation(emulated_library):
    t.check_host_dt_is_device_dt(t.taylor_green(8, 2, e0=1.0), 3)


def test_two_runs_bitwise_on_the_emulation(emulated_library):
    t.check_two_runs_bitwise(t.taylor_green(8, 2, e0=1.0), 3)


def test_dump_and_restart_on_the_emulation(emulated_library, tmp_path):
    t.check_dump_and_restart(t.taylor_green(8, 2, e0=1.0), 2, tmp_path)


def test_strided_layout_on_the_emulation(emulated_library):
    t.check_strided_layout(t.block(0.2, 2))
    t.check_strided_layout(t.block(0.34, 3, g=(0.0, 0.0, -9.81)))


def test_reproducing_property_on_the_emulation(emulated_library):
    t.check_reproducing(t.block(0.05, 2), 1e-6)


def test_momentum_conservation_on_the_emulation(emulated_library):
    t.check_momentum_conservation(t.taylor_green(10, 2, perturb=0.0, e0=1.0), 1e-12)


def test_refusals_on_the_emulation(emulated_library):
    t.check_refusals(t.block(0.25, 2))
    t.check_ghosts_1d_and_mirror_refused()


def test_property_ids_on_the_emulation(emulated_library):
    t.check_property_ids()
