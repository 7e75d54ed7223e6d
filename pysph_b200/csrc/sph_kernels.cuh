// sph_kernels.cuh -- the SPH smoothing kernels in fp32.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// SPH smoothing kernels in fp32 (pysph/base/kernels.py; see oracle for fp64)
//   returns w = W(q)/sigma-free value * fac  and  dw = dW/dq * fac
// --------------------------------------------------------------------------
template <int DIM> __device__ __forceinline__ float hpow(float h1)
{
    return DIM == 1 ? h1 : (DIM == 2 ? h1 * h1 : h1 * h1 * h1);
}

template <int K> __device__ __forceinline__ void sph_kernel(float q, float &w, float &dw);

// CubicSpline kernels.py:69-124, as clamped truncated powers (no compares, no selects): with
// t = clamp(1 - q/2, 0, 1) and s = clamp(1 - q, 0, 1), w = 2 t^3 - s^3 and dw = -3 min(q/2, t) (s + t)
// for every q >= 0 (q > 2 included).  The product form of dw equals 3 (s^2 - t^2) without its
// cancellation near q = 0.  The clamps compile to .SAT.
template <> __device__ __forceinline__ void sph_kernel<0>(float q, float &w, float &dw)
{
    const float hq = 0.5f * q;
    const float t = fminf(fmaxf(1.0f - hq, 0.0f), 1.0f);
    const float s = fminf(fmaxf(1.0f - q, 0.0f), 1.0f);
    w = 2.0f * (t * t * t) - s * s * s;
    dw = -3.0f * fminf(hq, t) * (s + t);
}
// WendlandQuintic kernels.py:304-343
template <> __device__ __forceinline__ void sph_kernel<1>(float q, float &w, float &dw)
{
    const float t = 1.0f - 0.5f * q;
    const float t3 = t * t * t;
    w = q < 2.0f ? t3 * t * (2.0f * q + 1.0f) : 0.0f;
    dw = q < 2.0f ? -5.0f * q * t3 : 0.0f;
}
// QuinticSpline kernels.py:1087-1153
template <> __device__ __forceinline__ void sph_kernel<2>(float q, float &w, float &dw)
{
    const float t3 = 3.0f - q, t2 = 2.0f - q, t1 = 1.0f - q;
    const float a3 = t3 * t3, a2 = t2 * t2, a1 = t1 * t1;
    const float p3 = a3 * a3, p2 = a2 * a2, p1 = a1 * a1;  // 4th powers
    float ww = 0.0f, dd = 0.0f;
    if (q <= 3.0f) { ww = p3 * t3; dd = -5.0f * p3; }
    if (q <= 2.0f) { ww -= 6.0f * p2 * t2; dd += 30.0f * p2; }
    if (q <= 1.0f) { ww += 15.0f * p1 * t1; dd -= 75.0f * p1; }
    w = ww;
    dw = dd;
}
// Gaussian kernels.py:864-898
template <> __device__ __forceinline__ void sph_kernel<3>(float q, float &w, float &dw)
{
    const float e = __expf(-q * q);
    w = q < 3.0f ? e : 0.0f;
    dw = q < 3.0f ? -2.0f * q * e : 0.0f;
}
