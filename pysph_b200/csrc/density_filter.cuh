// density_filter.cuh -- the density re-initialisation of DensityCorrection: ShepardFilter,
// MLSFirstOrder2D and MLSFirstOrder3D over the persistent neighbour lists.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// density re-initialisation (pysph/sph/wc/density_correction.py, pysph/solver/tools.py:97-205)
//
// initialize: rhotmp = rho.  loop_all: rho_i from the sources' rhotmp, the source array being
// the destination array itself; every value a destination reads is from before the filter
// (k_dfilter_pack takes them all before k_density_filter writes rho).
//   Shepard:  rho_i = sum m_j W_ij / sum (m_j / rhotmp_j) W_ij
//   MLS:      A = sum (m_j / rhotmp_j) W_ij p p^T, p = [1, x_ij, y_ij (, z_ij)]; A b = e0 solved
//             as gj_solve does (linalg.py:94-166); rho_i = sum m_j (b . p) W_ij
// W_ij with h_ij = (h_i + h_j) / 2 and the FILTER's kernel, which may differ from the
// evaluation's; the accept test is the neighbour search's with that kernel's radius scale.
// --------------------------------------------------------------------------
#define DFILTER_NT 128

struct DensityFilterArgs {
    const float4 *AB;          // the packed positions (x, y, z, h), cell-relative: A half of AB
    float4 *F;                 // [2 n] the filter's records: A, then (m, m / rhotmp, type bits, 0)
    const uint32_t *perm, *cnt, *lst;
    const uint8_t *stype;
    const double *m;
    double *rho, *rhotmp;
    long long n;
    int capg;
    float cellx, celly, cellz;
    float k2;                  // the filter kernel's radius_scale^2
    float kfac;                // ... and its normalisation for this dim
    unsigned mask;             // the arrays filtered
    int real_only;
};

// initialize (rhotmp = rho) of the filtered arrays, and the records the walks gather: one
// 32-byte sector per particle, like AB
__global__ void k_dfilter_pack(const DensityFilterArgs a)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const int t = a.stype[s];
    const uint32_t g = a.perm[s];
    const double m = a.m[g];
    float v = 0.0f;
    if ((a.mask >> (t & 7)) & 1u) {
        const double rt = a.rho[g];
        a.rhotmp[g] = rt;
        v = (float)(m / rt);
    }
    a.F[2 * s] = a.AB[2 * s];
    a.F[2 * s + 1] = make_float4((float)m, v, __int_as_float(t), 0.0f);
}

// gj_solve (linalg.py:94-166) on [A | B], NB right-hand-side columns, in its operation order.  Its
// pivot search swaps an element with itself, so this is elimination without pivoting.  false: one
// of its two early returns, which leave the caller's result as it was (the back substitution tests
// the last column only, as the reference does).
template <int N, int NB = 1> __device__ __forceinline__ bool gj_solve(double (&m)[N][N + NB])
{
#pragma unroll
    for (int c = 0; c < N; c++)
#pragma unroll
        for (int r = c + 1; r < N; r++) {
            const double d = m[c][c];
            if (fabs(d) < 1e-12) return false;
            const double cc = -m[r][c] / d;
#pragma unroll
            for (int j = 0; j < N + NB; j++) m[r][j] = m[r][j] + cc * m[c][j];
        }
#pragma unroll
    for (int rb = N - 1; rb >= 0; rb--) {
        if (m[rb][rb] == 0.0) {
            if (fabs(m[rb][N + NB - 1]) > 1e-12) return false;
        } else {
#pragma unroll
            for (int bc = N + NB - 1; bc >= rb; bc--) m[rb][bc] = m[rb][bc] / m[rb][rb];
#pragma unroll
            for (int ku = rb - 1; ku >= 0; ku--)
#pragma unroll
                for (int kl = N + NB - 1; kl >= rb; kl--) {
                    const double kk = -m[ku][rb] / m[rb][rb];
                    m[ku][kl] = m[ku][kl] + kk * m[rb][kl];
                }
        }
    }
    return true;
}

// One THREAD per destination walks its list (list_walk); MODE is a B200SPH_DFILTER_* id.  Shepard
// makes one walk; MLS makes two over the same list, the moments in the first, the fp64 solve
// between them.
template <int K, int DIM, int MODE>
__global__ void __launch_bounds__(DFILTER_NT) k_density_filter(const DensityFilterArgs a)
{
    constexpr int NP = MODE == B200SPH_DFILTER_MLS3D ? 4 : 3;   // MLS: the size of p
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * DFILTER_NT + threadIdx.x;
    bool active = s < a.n;
    float4 Ai = make_float4(0.f, 0.f, 0.f, 0.f);
    int ti = 0, count = 0;
    if (active) {
        ti = __float_as_int(a.F[2 * s + 1].z);
        if (!((a.mask >> (ti & 7)) & 1u) || (a.real_only && (ti & PT_GHOST))) active = false;
    }
    if (active) {
        Ai = a.F[2 * s];
        count = (int)a.cnt[s];
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *nxt = list_slot(a.lst, a.capg, s);
    const float hi2 = a.k2 * Ai.w * Ai.w;
    struct Rec { float4 A, B; };
    const auto load = [&](const uint32_t e, Rec &r) { ld_256(a.F + 2u * LIST_J(e), r.A, r.B); };
    // W_ij of a list entry, 0 unless the pair passes the exact accept test and the source is of
    // the destination's array (the lists may hold other arrays' entries for other passes)
    const auto weight = [&](const bool live, const uint32_t e, const Rec &r, float &xij, float &yij, float &zij) {
        const float r2 = list_dist(e, a.cellx, a.celly, a.cellz, Ai, r.A, xij, yij, zij);
        const bool take = live && NNPS_ACCEPT(r2, hi2, a.k2, r.A.w) && ((__float_as_int(r.B.z) & 7) == (ti & 7));
        const float rinv = r2 > 1e-24f ? frsqrt(r2) : 0.0f;      // RIJ > 1e-12 guard, kernels.py:128-132
        const float h1 = frcp(0.5f * (Ai.w + r.A.w));
        float w, dw;
        sph_kernel<K>(r2 * rinv * h1, w, dw);
        return take ? w * (a.kfac * hpow<DIM>(h1)) : 0.0f;
    };
    double rho_new = 0.0;
    if constexpr (MODE == B200SPH_DFILTER_SHEPARD) {
        float sm = 0.f, sv = 0.f;   // sum m_j W_ij, sum (m_j / rhotmp_j) W_ij
        list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
            float xij, yij, zij;
            const float w = weight(live, e, r, xij, yij, zij);
            sm = fmaf(r.B.x, w, sm);
            sv = fmaf(r.B.y, w, sv);
        });
        rho_new = (double)sm / (double)sv;
    } else {
        // the distinct entries of the symmetric A, row by row: (0,0) (0,1) .. (0,NP-1) (1,1) ..
        float mom[NP * (NP + 1) / 2];
#pragma unroll
        for (int k = 0; k < NP * (NP + 1) / 2; k++) mom[k] = 0.f;
        list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
            float xij, yij, zij;
            const float vw = r.B.y * weight(live, e, r, xij, yij, zij);
            const float p[4] = {1.0f, xij, yij, zij};
            int k = 0;
#pragma unroll
            for (int i = 0; i < NP; i++)
#pragma unroll
                for (int j = i; j < NP; j++, k++) mom[k] = fmaf(p[i] * p[j], vw, mom[k]);
        });
        double aug[NP][NP + 1];
        {
            int k = 0;
#pragma unroll
            for (int i = 0; i < NP; i++) {
#pragma unroll
                for (int j = i; j < NP; j++, k++) aug[i][j] = aug[j][i] = (double)mom[k];
                aug[i][NP] = i == 0 ? 1.0 : 0.0;
            }
        }
        float b[4] = {1.0f, 0.0f, 0.0f, 0.0f};
        if (gj_solve<NP>(aug)) {
#pragma unroll
            for (int i = 0; i < NP; i++) b[i] = (float)aug[i][NP];
        }
        float sr = 0.f;
        list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
            float xij, yij, zij;
            const float w = weight(live, e, r, xij, yij, zij);
            const float bp = b[0] + b[1] * xij + b[2] * yij + (NP == 4 ? b[3] * zij : 0.0f);
            sr = fmaf(r.B.x, bp * w, sr);
        });
        rho_new = (double)sr;
    }
    if (active) a.rho[a.perm[s]] = rho_new;
}
