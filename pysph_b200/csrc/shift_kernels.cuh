// shift_kernels.cuh -- particle shifting of ShiftPositions: SimpleShift, FickianShift and
// CorrectVelocities over the persistent neighbour lists.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// particle shifting (pysph/sph/wc/shift.py)
//
// Sources are the destination's own array, the particle itself included (the tool's
// SPHEvaluator holds that array only).  Every destination's dpos is formed from the positions
// before the shift and only then are the particles moved (a Jacobi update: the reference's
// loop_all writes d_x in place while later destinations read s_x).
//   SimpleShift   (shift.py:41-83)   dpos_i = beta ri^2 vmax dt sum x_ij / (r_ij^3 + 1e-8),
//                                    ri = mean r_ij over the accepted entries, vmax = max |v|
//   FickianShift  (shift.py:86-148)  dpos_i = -C h_i |v_i| dt sum V_j (1 + f_ij) grad W(x_ij, h_ij),
//                                    f_ij = R (W_ij / W(h_i / hdx, h_i))^n with tensile_correction
//   CorrectVelocities (shift.py:151-188), after the neighbour search has seen the new positions:
//                                    gradv[3 b + a] = -sum V_j v_ij[a] DW_ij[b],
//                                    u_i[k] += sum_l gradv[3 k + l] dpos_i[l]
//                                    (as written, the TRANSPOSE of grad v applied to dpos)
// The records hold the pool's fp64 positions, so x_ij, r^2 and the accept test are formed in
// fp64 (the neighbour set of SimpleShift's unweighted sum jumps at the accept radius); the
// image shift of a periodic neighbour comes from the list entry's cell offset, and the image
// is x_j +- L, as a materialised ghost would be.  The sums are fp64; the kernel values are
// sph_kernel<K> in fp32.  dpos and the velocity change are indexed by pool index (gid), not by
// sorted slot: the neighbour-search update between the shift and the correction may re-sort.
// --------------------------------------------------------------------------
#define SHIFT_NT 128

struct ShiftRec { double x, y, z, w; };   // (x, y, z, h) or (u, v, w, m / rho): 32 bytes

struct ShiftArgs {
    ShiftRec *P, *V;                 // [n] by sorted slot (k_shift_pack)
    const uint32_t *perm, *cnt, *lst, *skey;
    const uint8_t *stype;
    double *x, *y, *z, *u, *v, *w;   // the pool
    const double *h, *m, *rho;
    double *dpos;                    // [3 pool] dpos by gid
    double *dvel;                    // [3 pool] CorrectVelocities' change of (u, v, w) by gid
    long long *vmax;                 // [B200SPH_MAX_ARRAYS] the bits of max |v| per array (>= 0)
    unsigned long long *pair_counter;  // the accepted entries (N_NBRS summed), or null
    long long n;
    int capg;
    int ncx, ncy, zorder;
    int per[3];                      // periodic axes
    double L[3];                     // the periodic box
    double kr;                       // the kernel's radius scale
    double kfac;                     // ... and its normalisation for this dim
    unsigned mask;                   // the arrays shifted / corrected
    double dt, coef;                 // the tool's dt; beta (simple) or C (fickian)
    double hdx, tR, tn;              // FickianShift's hdx, tensile_const, tensile_pow
    int tensile;
};

// fp64 products and sums as written (no contraction into FMA), so that r^2 and the accept test
// are those of the reference's fp64 loop
__device__ __forceinline__ double shift_mul(const double a, const double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__device__ __forceinline__ double shift_add(const double a, const double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// the records the walks gather, one pair of 32-byte records per sorted slot
__global__ void k_shift_pack(const ShiftArgs a)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const uint32_t g = a.perm[s];
    a.P[s] = ShiftRec{a.x[g], a.y[g], a.z[g], a.h[g]};
    a.V[s] = ShiftRec{a.u[g], a.v[g], a.w[g], a.m[g] / a.rho[g]};
}

// SimpleShift.py_initialize: max |v| over the pool range [off, off + n) of one array, into
// *out (zeroed before).  |v| >= 0, so its bits order like signed integers.
__global__ void k_shift_vmax(const double *__restrict__ u, const double *__restrict__ v, const double *__restrict__ w,
                             const long long off, const long long n, long long *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double vm = 0.0;
    if (i < n) {
        const double ui = u[off + i], vi = v[off + i], wi = w[off + i];
        vm = sqrt(shift_add(shift_add(shift_mul(ui, ui), shift_mul(vi, vi)), shift_mul(wi, wi)));
    }
    for (int o = 16; o > 0; o >>= 1) vm = fmax(vm, __shfl_xor_sync(0xffffffffu, vm, o));
    if ((threadIdx.x & 31) == 0 && vm > 0.0) atomicMax(out, __double_as_longlong(vm));
}

// (these three helpers take any argument block with the ShiftArgs geometry fields: the IISPH
// passes share them)
// x_ij = x_i - (x_j + image) of list entry e in fp64 and r^2 as the reference forms them.  The
// entry's cell offset d puts the source in the apparent cell c_i + d; where that differs from
// its own cell of the build (a periodic wrap), the image is the source shifted by the box.
template <class A>
__device__ __forceinline__ double shift_dist(const A &a, const uint32_t e, const ShiftRec &Pi, const ShiftRec &Pj,
                                             const uint32_t ci[3], const uint32_t keyj, double xij[3])
{
    uint32_t cj[3];
    grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, keyj, cj[0], cj[1], cj[2]);
    const double xi[3] = {Pi.x, Pi.y, Pi.z}, xj[3] = {Pj.x, Pj.y, Pj.z};
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const int app = (int)ci[d] + (int)((e >> (2 * d)) & 3u) - 1;
        double s = xj[d];
        if (a.per[d] && app != (int)cj[d]) s = shift_add(s, app > (int)cj[d] ? a.L[d] : -a.L[d]);
        xij[d] = shift_add(xi[d], -s);
    }
    return shift_add(shift_add(shift_mul(xij[0], xij[0]), shift_mul(xij[1], xij[1])), shift_mul(xij[2], xij[2]));
}

// linked_list_nnps.pyx:188 in fp64: r^2 < (k h_i)^2 or r^2 < (k h_j)^2
template <class A>
__device__ __forceinline__ bool shift_accept(const A &a, const double r2, const double hi, const double hj)
{
    const double ki = shift_mul(a.kr, hi), kj = shift_mul(a.kr, hj);
    return r2 < shift_mul(ki, ki) || r2 < shift_mul(kj, kj);
}

// W(r, h) and grad W(x, r, h) (kernels.py) with the kernel polynomial in fp32
template <int K, int DIM, class A>
__device__ __forceinline__ void shift_kernel(const A &a, const double xij[3], const double rij, const double hij,
                                             double &wij, double dwij[3])
{
    const double h1 = 1.0 / hij;
    float w, dw;
    sph_kernel<K>((float)(rij * h1), w, dw);
    const double fac = a.kfac * (DIM == 1 ? h1 : (DIM == 2 ? h1 * h1 : h1 * h1 * h1));
    wij = fac * (double)w;
    const double tmp = rij > 1e-12 ? fac * (double)dw * h1 / rij : 0.0;   // kernels.py:128-132
#pragma unroll
    for (int d = 0; d < 3; d++) dwij[d] = tmp * xij[d];
}

// the destination of slot s, or false: not of the arrays in a.mask, or a ghost
__device__ __forceinline__ bool shift_dest(const ShiftArgs &a, const long long s, int &ti)
{
    if (s >= a.n) return false;
    ti = a.stype[s];
    return ((a.mask >> (ti & 7)) & 1u) && !(ti & PT_GHOST);
}

// One THREAD per destination walks its list (list_walk); dpos -> a.dpos[3 gid].  KIND is a
// B200SPH_SHIFT_* id.  Nothing is moved here (k_shift_apply does that after every dpos is known).
template <int K, int DIM, int KIND>
__global__ void __launch_bounds__(SHIFT_NT) k_shift(const ShiftArgs a)
{
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * SHIFT_NT + threadIdx.x;
    int ti = 0, count = 0;
    const bool active = shift_dest(a, s, ti);
    ShiftRec Pi = {0.0, 0.0, 0.0, 0.0}, Vi = Pi;
    uint32_t ci[3] = {0u, 0u, 0u};
    if (active) {
        Pi = a.P[s];
        Vi = a.V[s];
        count = (int)a.cnt[s];
        grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, a.skey[s], ci[0], ci[1], ci[2]);
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *nxt = list_slot(a.lst, a.capg, s);
    struct Rec { ShiftRec P; double Vj; uint32_t key; int t; };
    const auto load = [&](const uint32_t e, Rec &r) {
        const uint32_t j = LIST_J(e);
        r.P = a.P[j];
        if (KIND == B200SPH_SHIFT_FICKIAN) r.Vj = a.V[j].w;
        r.key = a.skey[j];
        r.t = a.stype[j];
    };
    double sum[3] = {0.0, 0.0, 0.0}, ri = 0.0;
    int nnbrs = 0;
    // FickianShift: W(h_i / hdx, h_i), the reference of the tensile correction
    double wdx = 0.0;
    if (KIND == B200SPH_SHIFT_FICKIAN && a.tensile) {
        const double dx[3] = {Pi.w / a.hdx, 0.0, 0.0};
        double dw[3];
        shift_kernel<K, DIM>(a, dx, dx[0], Pi.w, wdx, dw);
    }
    list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
        if (!live || (r.t & 7) != (ti & 7)) return;
        double xij[3];
        const double r2 = shift_dist(a, e, Pi, r.P, ci, r.key, xij);
        if (!shift_accept(a, r2, Pi.w, r.P.w)) return;
        const double rij = sqrt(r2);
        nnbrs++;
        if constexpr (KIND == B200SPH_SHIFT_SIMPLE) {
            const double r3 = rij * rij * rij + 1.0e-08;
#pragma unroll
            for (int d = 0; d < 3; d++) sum[d] += xij[d] / r3;
            ri += rij;
        } else {
            double wij, dwij[3];
            shift_kernel<K, DIM>(a, xij, rij, (Pi.w + r.P.w) * 0.5, wij, dwij);
            const double fij = a.tensile ? a.tR * pow(wij / wdx, a.tn) : 0.0;
            const double f = r.Vj * (1.0 + fij);
#pragma unroll
            for (int d = 0; d < 3; d++) sum[d] += f * dwij[d];
        }
    });
    pairs_flush(a, (unsigned)nnbrs);
    if (!active) return;
    double fac;
    if constexpr (KIND == B200SPH_SHIFT_SIMPLE) {
        ri = ri / nnbrs;
        fac = a.coef * ri * ri * __longlong_as_double(a.vmax[ti & 7]) * a.dt;
    } else {
        const double vmag = sqrt(Vi.x * Vi.x + Vi.y * Vi.y + Vi.z * Vi.z);
        fac = -a.coef * Pi.w * vmag * a.dt;
    }
    const uint32_t g = a.perm[s];
#pragma unroll
    for (int d = 0; d < 3; d++) a.dpos[3 * (size_t)g + d] = fac * sum[d];
}

// CorrectVelocities: the change of (u, v, w) -> a.dvel[3 gid], from the velocities before it
template <int K, int DIM>
__global__ void __launch_bounds__(SHIFT_NT) k_correct_velocities(const ShiftArgs a)
{
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * SHIFT_NT + threadIdx.x;
    int ti = 0, count = 0;
    const bool active = shift_dest(a, s, ti);
    ShiftRec Pi = {0.0, 0.0, 0.0, 0.0}, Vi = Pi;
    uint32_t ci[3] = {0u, 0u, 0u};
    if (active) {
        Pi = a.P[s];
        Vi = a.V[s];
        count = (int)a.cnt[s];
        grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, a.skey[s], ci[0], ci[1], ci[2]);
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *nxt = list_slot(a.lst, a.capg, s);
    struct Rec { ShiftRec P, V; uint32_t key; int t; };
    const auto load = [&](const uint32_t e, Rec &r) {
        const uint32_t j = LIST_J(e);
        r.P = a.P[j];
        r.V = a.V[j];
        r.key = a.skey[j];
        r.t = a.stype[j];
    };
    double gradv[9];
#pragma unroll
    for (int k = 0; k < 9; k++) gradv[k] = 0.0;
    unsigned npairs = 0;
    list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
        if (!live || (r.t & 7) != (ti & 7)) return;
        double xij[3];
        const double r2 = shift_dist(a, e, Pi, r.P, ci, r.key, xij);
        if (!shift_accept(a, r2, Pi.w, r.P.w)) return;
        npairs++;
        double wij, dwij[3];
        shift_kernel<K, DIM>(a, xij, sqrt(r2), (Pi.w + r.P.w) * 0.5, wij, dwij);
        const double vij[3] = {Vi.x - r.V.x, Vi.y - r.V.y, Vi.z - r.V.z};
#pragma unroll
        for (int al = 0; al < 3; al++)
#pragma unroll
            for (int be = 0; be < 3; be++) gradv[3 * be + al] += -r.V.w * vij[al] * dwij[be];
    });
    pairs_flush(a, npairs);
    if (!active) return;
    const uint32_t g = a.perm[s];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double tmp = 0.0;
#pragma unroll
        for (int j = 0; j < 3; j++) tmp += gradv[3 * i + j] * a.dpos[3 * (size_t)g + j];
        a.dvel[3 * (size_t)g + i] = tmp;
    }
}

// q[gid] += d[3 gid + 0..2] for the destinations of a walk over the same sorted order: moves the
// particles by dpos after k_shift, or corrects their velocities after k_correct_velocities
__global__ void k_shift_apply(const ShiftArgs a, const double *__restrict__ d, double *q0, double *q1, double *q2)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int ti = 0;
    if (!shift_dest(a, s, ti)) return;
    const size_t g = a.perm[s];
    q0[g] += d[3 * g];
    q1[g] += d[3 * g + 1];
    q2[g] += d[3 * g + 2];
}
