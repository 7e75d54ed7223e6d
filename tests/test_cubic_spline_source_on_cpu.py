"""sph_kernel<0> (CubicSpline, pysph_b200/csrc/sph_kernels.cuh) extracted verbatim from the
library source, compiled for the host and evaluated in fp32 on a dense q grid against the fp64
piecewise form of kernels.py:69-124: q -> 0, both sides of q = 1 and q = 2, and q > 2, where
w and dw must be exactly 0.  The fp32 form is the clamped truncated powers, with no compares
and no selects; this pins it to the piecewise polynomials."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pysph_b200.build import read_source

HEAD = 'template <> __device__ __forceinline__ void sph_kernel<0>('

SHIM = r'''
#include <cmath>
#define __device__
#define __forceinline__ inline
template <int K> void sph_kernel(float q, float &w, float &dw);
%s
extern "C" void cubic_spline(const float *q, float *w, float *dw, long n)
{
    for (long i = 0; i < n; i++) sph_kernel<0>(q[i], w[i], dw[i]);
}
'''


def _extract():
    src = read_source().split('\n')
    i = next(k for k, ln in enumerate(src) if ln.startswith(HEAD))
    j = next(k for k in range(i, len(src)) if src[k] == '}')
    return '\n'.join(src[i:j + 1])


@pytest.fixture(scope='module')
def spline(tmp_path_factory):
    d = tmp_path_factory.mktemp('cubic_spline')
    cpp, so = os.path.join(d, 'spline.cpp'), os.path.join(d, 'spline.so')
    with open(cpp, 'w') as f:
        f.write(SHIM % _extract())
    cxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.check_call([cxx, '-O1', '-std=c++17', '-shared', '-fPIC', '-ffp-contract=off',
                           cpp, '-o', so])
    lib = C.CDLL(so)

    def run(q):
        q = np.ascontiguousarray(q, dtype=np.float32)
        w, dw = np.empty_like(q), np.empty_like(q)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        lib.cubic_spline(p(q), p(w), p(dw), C.c_long(q.size))
        return w, dw
    return run


def _reference(q):
    q = q.astype(np.float64)
    t2 = 2.0 - q
    w = np.where(q > 2, 0.0, np.where(q > 1, 0.25 * t2 ** 3, 1 - 1.5 * q * q * (1 - 0.5 * q)))
    dw = np.where(q > 2, 0.0, np.where(q > 1, -0.75 * t2 ** 2, -3 * q * (1 - 0.75 * q)))
    return w, dw


def test_cubic_spline_source_vs_fp64(spline):
    f = np.float32
    edges = []      # q -> 0 by normal numbers only: q >= 1e-12 / h for r >= 1e-12 (RIJ guard)
    for x in (f(1), f(2)):
        y = x
        for _ in range(4):
            y = np.nextafter(y, f(3))
            edges.append(y)
        y = x
        for _ in range(4):
            y = np.nextafter(y, f(-1))
            edges.append(y)
    q = np.concatenate([np.linspace(0, 2.5, 500001, dtype=np.float32),
                        np.array(edges, dtype=np.float32),
                        np.array([0, 1e-30, 1e-12, 1e-6, 1e-3, 1, 2, 2.0001, 3, 1e3, 1e30],
                                 dtype=np.float32)])
    q = q[q >= 0]
    w, dw = spline(q)
    wr, dwr = _reference(q)
    assert np.max(np.abs(w - wr)) <= 5e-7
    nz = dwr != 0
    assert np.max(np.abs(dw[nz] - dwr[nz]) / np.abs(dwr[nz])) <= 2e-7
    out = q >= 2
    assert out.sum() > 1000
    assert np.all(w[out] == 0) and np.all(dw[out] == 0)
    assert w[q == 0][0] == 1 and dw[q == 0][0] == 0
