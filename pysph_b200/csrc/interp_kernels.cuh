// interp_kernels.cuh -- PySPH's Interpolator (pysph/tools/interpolator.py:18-172): particle
// fields at arbitrary probe points.  Part of the single translation unit b200sph.cu (included
// there, in this order; not a stand-alone header).
//
// A probe is not a particle: no neighbour list serves it.  One WARP per probe walks the cells of
// the context's last build that lie within reach, its lanes over the particles of a cell.  The
// build's sorted order and cells are used as they are, whatever the particles did since: a
// particle of cell c lies within D_d of c's box along axis d, D_d measured over every source by
// k_interp_pack in the same pass that packs the records, so the cells whose box grown by
// reach + D_d meets the probe hold every source within reach (DESIGN.md, "Interpolator").
//   shepard      sum W_ij f_j / sum W_ij            (the division only when the sum > 1e-12)
//   sph          sum (m/rho)_j W_ij f_j
//   splash       sum (m/rho)_j WI f_j               (WI: W at h_p)
//   splash_norm  sum (m/rho)_j WJ f_j / sum (m/rho)_j WJ, the same guard   (WJ: W at h_j)
//   order1       SPHFirstOrderApproximationPreStep + SPHFirstOrderApproximation: the moments and
//                p_sph, then augmented_matrix + gj_solve with n = dim + 1 (value, gradient);
//                rho_j is SummationDensity over the sources first (k_interp_density)
// W_ij at h_ij = (h_p + h_j) / 2; the accept test is the neighbour search's,
// r^2 < (k h_p)^2 or r^2 < (k h_j)^2, k the interpolation kernel's radius scale.
// --------------------------------------------------------------------------
#define INTERP_NT 128

struct InterpArgs {
    const double *x, *y, *z, *h, *m, *rho;    // the pool, by pool index
    const double *fd[B200SPH_MAX_ARRAYS];     // the interpolated property per array: fp64 ...
    const float *ff[B200SPH_MAX_ARRAYS];      // ... or fp32; both null: the array lacks it (f = 0)
    const uint32_t *perm, *skey, *cell_start;
    const uint8_t *stype;
    long long n;                              // sorted particles
    GridDev G;                                // the build's grid
    float4 *Q;                                // [2 n]: (x, y, z relative to the build cell, h), (f, m, rho, type; -1: not a source)
    float *rho_sph;                           // [n] order1: SummationDensity of the sources
    unsigned *red;                            // [0..2] D_d, [3] max h of the sources (float bits); [4] 1: a stencil wrapped onto itself
    unsigned mask;                            // the source arrays
    const double *px, *py, *pz;               // the probes
    long long np;
    float hp;                                 // the probes' h
    float k;                                  // the kernel's radius scale ...
    float kfac;                               // ... and its normalisation for dim
    int method;                               // B200SPH_INTERP_*
    double *out;                              // [np], order1 [4 np]
};

// the records the walks gather, one 32-byte sector per particle, and the reach of the stencil
__global__ void k_interp_pack(const InterpArgs a)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float ox = 0.f, oy = 0.f, oz = 0.f, hm = 0.f;
    if (s < a.n) {
        const uint32_t g = a.perm[s];
        const int t = a.stype[s];
        const int arr = t & 7;
        const float4 P = pack_position(a.G, a.skey[s], a.x[g], a.y[g], a.z[g], a.h[g]);
        const bool src = (a.mask >> arr) & 1u;
        float f = 0.f;
        if (src && a.fd[arr]) f = (float)a.fd[arr][g];
        else if (src && a.ff[arr]) f = a.ff[arr][g];
        a.Q[2 * s] = P;
        a.Q[2 * s + 1] = make_float4(f, (float)a.m[g], (float)a.rho[g], __int_as_float(src ? t : -1));
        if (src) {
            ox = fmaxf(fmaxf(-P.x, P.x - (float)a.G.cell[0]), 0.f);
            oy = fmaxf(fmaxf(-P.y, P.y - (float)a.G.cell[1]), 0.f);
            oz = fmaxf(fmaxf(-P.z, P.z - (float)a.G.cell[2]), 0.f);
            hm = P.w;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ox = fmaxf(ox, __shfl_xor_sync(0xffffffffu, ox, o));
        oy = fmaxf(oy, __shfl_xor_sync(0xffffffffu, oy, o));
        oz = fmaxf(oz, __shfl_xor_sync(0xffffffffu, oz, o));
        hm = fmaxf(hm, __shfl_xor_sync(0xffffffffu, hm, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (ox > 0.f) atomicMax(&a.red[0], __float_as_uint(ox));
        if (oy > 0.f) atomicMax(&a.red[1], __float_as_uint(oy));
        if (oz > 0.f) atomicMax(&a.red[2], __float_as_uint(oz));
        if (hm > 0.f) atomicMax(&a.red[3], __float_as_uint(hm));
    }
}

// The cells within reach of q (fp64, wrapped into a periodic box as _box_wrap_periodic does,
// nnps_base.pyx:699-743), each visited once per image; `body(t, R, S, xij, yij, zij)` per lane
// and sorted particle t of a cell (S.w = -1 past the cell's end).  Warp-uniform: every lane of the warp passes the same q and reach.
template <class F>
__device__ __forceinline__ void interp_walk(const InterpArgs &a, double q[3], const float reach, F &&body)
{
    const GridDev &G = a.G;
    int lo[3], hi[3];
    bool self_wrap = false;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const double L = G.cell[d] * G.nc[d];
        if (G.periodic[d]) {
            if (q[d] < G.xmin[d]) q[d] += L;
            if (q[d] > G.xmin[d] + L) q[d] -= L;
        }
        // (the fp32 measurements of D and h get a relative margin)
        const double r = 1.0001 * ((double)reach + (double)__uint_as_float(a.red[d])) + 1e-6 * G.cell[d];
        const double l = fmin(fmax(floor((q[d] - r - G.xmin[d]) / G.cell[d]), -1e9), 1e9);
        const double u = fmin(fmax(floor((q[d] + r - G.xmin[d]) / G.cell[d]), -1e9), 1e9);
        lo[d] = (int)l, hi[d] = (int)u;
        if (G.periodic[d]) {
            if (hi[d] - lo[d] + 1 > G.nc[d]) self_wrap = true, hi[d] = lo[d] + G.nc[d] - 1;
        } else {
            lo[d] = max(lo[d], 0), hi[d] = min(hi[d], G.nc[d] - 1);
        }
    }
    if (self_wrap && (threadIdx.x & 31) == 0) atomicMax(&a.red[4], 1u);
    const int lane = threadIdx.x & 31;
    for (int cz = lo[2]; cz <= hi[2]; cz++) {
        const int wz = G.periodic[2] ? ((cz % G.nc[2]) + G.nc[2]) % G.nc[2] : cz;
        const float qz = (float)(q[2] - (G.xmin[2] + (double)cz * G.cell[2]));
        for (int cy = lo[1]; cy <= hi[1]; cy++) {
            const int wy = G.periodic[1] ? ((cy % G.nc[1]) + G.nc[1]) % G.nc[1] : cy;
            const float qy = (float)(q[1] - (G.xmin[1] + (double)cy * G.cell[1]));
            const uint32_t row = (uint32_t)G.nc[0] * grid_row(G.zorder, (uint32_t)G.nc[1], (uint32_t)wy, (uint32_t)wz);
            for (int cx = lo[0]; cx <= hi[0]; cx++) {
                const int wx = G.periodic[0] ? ((cx % G.nc[0]) + G.nc[0]) % G.nc[0] : cx;
                const float qx = (float)(q[0] - (G.xmin[0] + (double)cx * G.cell[0]));
                const uint32_t key = row + (uint32_t)wx;
                const uint32_t rs = a.cell_start[key], re = a.cell_start[key + 1];
                for (uint32_t t0 = rs; t0 < re; t0 += 32) {
                    const uint32_t t = t0 + lane;
                    float4 R = make_float4(0.f, 0.f, 0.f, 0.f), S = make_float4(0.f, 0.f, 0.f, __int_as_float(-1));
                    if (t < re) ld_256(a.Q + 2u * t, R, S);
                    body(t, R, S, qx - R.x, qy - R.y, qz - R.z);
                }
            }
        }
    }
}

// order1's first Group: SummationDensity(dest = a, sources = every array) for every particle
// of the source arrays, ghosts included (Group real=False), into rho_sph -- never the pool's rho
template <int K, int DIM>
__global__ void __launch_bounds__(INTERP_NT) k_interp_density(const InterpArgs a)
{
    const long long s = ((long long)blockIdx.x * INTERP_NT + threadIdx.x) >> 5;
    const auto warp_sum = [](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    if (s >= a.n) return;
    const float4 Si = a.Q[2 * s + 1];
    if (__float_as_int(Si.w) < 0) return;
    const uint32_t g = a.perm[s];
    double q[3] = {a.x[g], a.y[g], a.z[g]};
    const float hi = a.Q[2 * s].w, k2 = a.k * a.k;
    const float reach = a.k * fmaxf(hi, __uint_as_float(a.red[3]));
    float sum = 0.f;
    interp_walk(a, q, reach, [&](const uint32_t, const float4 &R, const float4 &S, const float xij, const float yij, const float zij) {
        const float r2 = xij * xij + yij * yij + zij * zij;
        if (__float_as_int(S.w) < 0 || !(r2 < k2 * hi * hi || r2 < k2 * R.w * R.w)) return;
        const float h1 = frcp(0.5f * (hi + R.w));
        const float rinv = r2 > 1e-24f ? frsqrt(r2) : 0.0f;
        float w, dw;
        sph_kernel<K>(r2 * rinv * h1, w, dw);
        sum = fmaf(S.y, w * (a.kfac * hpow<DIM>(h1)), sum);
    });
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) a.rho_sph[s] = sum;
}

// the probes: one warp per probe
template <int K, int DIM, bool ORDER1>
__global__ void __launch_bounds__(INTERP_NT) k_interp(const InterpArgs a)
{
    const long long p = ((long long)blockIdx.x * INTERP_NT + threadIdx.x) >> 5;
    const auto warp_sum = [](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    if (p >= a.np) return;
    double q[3] = {a.px[p], a.py[p], a.pz[p]};
    const float hp = a.hp, k2 = a.k * a.k, hp2 = k2 * hp * hp;
    const float reach = a.k * fmaxf(hp, __uint_as_float(a.red[3]));
    const int method = a.method;
    const bool lane0 = (threadIdx.x & 31) == 0;
    if constexpr (!ORDER1) {
        float sw = 0.f, sf = 0.f;   // the weights (shepard, splash_norm) and the weighted values
        interp_walk(a, q, reach, [&](const uint32_t, const float4 &R, const float4 &S, const float xij, const float yij, const float zij) {
            const float r2 = xij * xij + yij * yij + zij * zij;
            if (__float_as_int(S.w) < 0 || !(r2 < hp2 || r2 < k2 * R.w * R.w)) return;
            const float hk = method == B200SPH_INTERP_SPLASH ? hp : (method == B200SPH_INTERP_SPLASH_NORM ? R.w : 0.5f * (hp + R.w));
            const float h1 = frcp(hk);
            const float rinv = r2 > 1e-24f ? frsqrt(r2) : 0.0f;
            float w, dw;
            sph_kernel<K>(r2 * rinv * h1, w, dw);
            w *= a.kfac * hpow<DIM>(h1);
            const float c = method == B200SPH_INTERP_SHEPARD ? w : S.y / S.z * w;
            sw += c;
            sf = fmaf(c, S.x, sf);
        });
        sw = warp_sum(sw);
        sf = warp_sum(sf);
        if (lane0) {
            double v = (double)sf;
            if ((method == B200SPH_INTERP_SHEPARD || method == B200SPH_INTERP_SPLASH_NORM) && (double)sw > 1e-12) v = v / (double)sw;
            a.out[p] = v;
        }
    } else {
        constexpr int N = DIM + 1;
        float mom[N][N], ps[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            ps[i] = 0.f;
#pragma unroll
            for (int j = 0; j < N; j++) mom[i][j] = 0.f;
        }
        interp_walk(a, q, reach, [&](const uint32_t t, const float4 &R, const float4 &S, const float xij, const float yij, const float zij) {
            const float r2 = xij * xij + yij * yij + zij * zij;
            if (__float_as_int(S.w) < 0 || !(r2 < hp2 || r2 < k2 * R.w * R.w)) return;
            const float h1 = frcp(0.5f * (hp + R.w));
            const float rinv = r2 > 1e-24f ? frsqrt(r2) : 0.0f;
            float w, dw;
            sph_kernel<K>(r2 * rinv * h1, w, dw);
            const float fh = a.kfac * hpow<DIM>(h1);
            const float V = S.y / a.rho_sph[t];
            const float WV = w * fh * V, GV = dw * fh * h1 * rinv * V;   // WIJ Vj, |DWIJ| Vj / rij
            const float X[3] = {xij, yij, zij};
            // row 0: W V, -X W V; row 1 + d: DW_d V, -X DW_d V (SPHFirstOrderApproximationPreStep)
            mom[0][0] += WV;
            ps[0] = fmaf(S.x, WV, ps[0]);
#pragma unroll
            for (int j = 1; j < N; j++) mom[0][j] -= X[j - 1] * WV;
#pragma unroll
            for (int i = 1; i < N; i++) {
                const float dv = GV * X[i - 1];
                mom[i][0] += dv;
                ps[i] = fmaf(S.x, dv, ps[i]);
#pragma unroll
                for (int j = 1; j < N; j++) mom[i][j] -= X[j - 1] * dv;
            }
        });
        double aug[N][N + 1];
#pragma unroll
        for (int i = 0; i < N; i++) {
#pragma unroll
            for (int j = 0; j < N; j++) aug[i][j] = (double)warp_sum(mom[i][j]);
            aug[i][N] = (double)warp_sum(ps[i]);
        }
        if (lane0) {
            const bool ok = gj_solve<N>(aug);   // its early return leaves the result at 0
#pragma unroll
            for (int i = 0; i < 4; i++) a.out[4 * p + i] = (ok && i < N) ? aug[i][N] : 0.0;
        }
    }
}
