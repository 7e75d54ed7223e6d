// iisph_kernels.cuh -- implicit incompressible SPH: the Groups of IISPHScheme.get_equations
// (pysph/sph/iisph.py:511-643) over the persistent neighbour lists, and IISPHStep.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).
//
// One THREAD per destination walks its list (list_walk) and keeps the sources of the arrays the
// pass reads; the geometry is the particle shifting's (shift_dist, shift_accept, shift_kernel):
// x_ij, r^2 and the accept test in fp64, a periodic image from the entry's cell offset, the
// kernel polynomial in fp32 and every sum in fp64.  A pass boundary lies wherever a body reads a
// source value the same Group writes:
//   IISPH_V      NumberDensity (:37-42), every solid over itself
//   IISPH_RHO    SummationDensity + SummationDensityBoundary (:45-59)
//   IISPH_ADV    AdvectionAcceleration + ComputeDII(+Boundary) + ViscosityAcceleration(+Boundary)
//                (:79-160); post-loop uadv = u + dt a
//   IISPH_AII    ComputeRhoAdvection + ComputeAII (+ ComputeRhoBoundary, ComputeAIIBoundary)
//                (:163-225); initialize rho_adv = rho, p0 = p, piter = 0.5 p
//   IISPH_DIJPJ  ComputeDIJPJ (:228-240), once per iteration
//   IISPH_SOLVE  PressureSolve(+Boundary) (:264-355) of ONE destination array, once per
//                iteration: the new pressure goes to pnext, k_iisph_commit copies it into
//                piter and p after every destination of that array has read the old piter (the
//                reference runs the loops of a destination before its post-loop); the next
//                array then sees it, as the reference's next destination does
//   IISPH_FORCE  PressureForce(+Boundary) (:367-402): au (initialize zeroes it: gravity and
//                viscosity reach the stepper through uadv only), dt_cfl = 2 |uadv|,
//                dt_force = 2 |a|^2
// The iterations run on the device: after each, k_iisph_partials / k_iisph_converge reduce
// PressureSolve.reduce's two sums of every fluid in a fixed order (no float atomics) and set
// IisphState::done when Group(iterate=True, min_iterations, max_iterations)'s condition
// (acceleration_eval_cython_helper.py:329-340) holds.  The host enqueues max_iterations
// iterations without waiting; the kernels of an iteration after `done` return at once.
// --------------------------------------------------------------------------
#define IISPH_NT 128
#define IISPH_RED 256     // threads (and elements per thread: 1) of a partial-sum block

enum { IISPH_V = 0, IISPH_RHO, IISPH_ADV, IISPH_AII, IISPH_DIJPJ, IISPH_SOLVE, IISPH_FORCE };

// the iteration state of the last evaluation (device memory)
struct IisphState {
    int it;            // iterations run
    int done;          // the iteration condition held: later iterations return at once
    int pad[2];
    double comp[B200SPH_MAX_ARRAYS];   // PressureSolve.compression of each fluid after `it`
};

struct IisphArgs {
    ShiftRec *P;                      // [n] (x, y, z, h) by sorted slot (k_iisph_pack)
    const uint32_t *perm, *cnt, *lst, *skey;
    const uint8_t *stype;
    const double *x, *y, *z, *h, *m, *rho_c;   // (rho_c: rho for the passes that read it)
    double *rho, *u, *v, *w, *V;
    double *uadv, *vadv, *wadv, *rho_adv, *dii0, *dii1, *dii2, *aii, *dijpj0, *dijpj1, *dijpj2;
    double *p, *p0, *piter, *pnext, *comp;
    float *au, *av, *aw, *dt_cfl, *dt_force;
    IisphState *st;
    double *part;                     // [2 nb] partial sums of one fluid: count, compression
    unsigned long long *pair_counter;
    long long n;
    int capg;
    int ncx, ncy, zorder;
    int per[3];
    double L[3];
    double kr, kfac;
    unsigned fluid_mask, solid_mask, dest_mask;
    double rho0, nu, gx, gy, gz, omega, tol;
    int min_it, max_it;
    double dt;
    const double *tc;                 // device-resident dt (tc[0]); null: dt
};

__device__ __forceinline__ double iisph_dt(const IisphArgs &a) { return a.tc ? a.tc[0] : a.dt; }

// the destination of slot s for a pass whose destinations are the arrays of `mask`
__device__ __forceinline__ bool iisph_dest(const IisphArgs &a, const long long s, const unsigned mask, int &ti)
{
    if (s >= a.n) return false;
    ti = a.stype[s];
    return ((mask >> (ti & 7)) & 1u) && !(ti & PT_GHOST);
}

__global__ void k_iisph_pack(const IisphArgs a)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const uint32_t g = a.perm[s];
    a.P[s] = ShiftRec{a.x[g], a.y[g], a.z[g], a.h[g]};
}

// a.st->done set: the iterations are over
__device__ __forceinline__ bool iisph_over(const IisphArgs &a, const int pass)
{
    return (pass == IISPH_DIJPJ || pass == IISPH_SOLVE) && *(volatile const int *)&a.st->done;
}

template <int K, int DIM, int PASS>
__global__ void __launch_bounds__(IISPH_NT) k_iisph(const IisphArgs a)
{
    if (iisph_over(a, PASS)) return;
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * IISPH_NT + threadIdx.x;
    const unsigned dmask = PASS == IISPH_V ? a.solid_mask : (PASS == IISPH_SOLVE ? a.dest_mask : a.fluid_mask);
    int ti = 0, count = 0;
    const bool active = iisph_dest(a, s, dmask, ti);
    ShiftRec Pi = {0.0, 0.0, 0.0, 0.0};
    uint32_t ci[3] = {0u, 0u, 0u}, gi = 0;
    double rhoi = 1.0, mi = 0.0, ui[3] = {0.0, 0.0, 0.0}, di[3] = {0.0, 0.0, 0.0}, dpi[3] = {0.0, 0.0, 0.0}, pi = 0.0;
    if (active) {
        Pi = a.P[s];
        count = (int)a.cnt[s];
        grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, a.skey[s], ci[0], ci[1], ci[2]);
        gi = a.perm[s];
        mi = a.m[gi];
        if (PASS != IISPH_V && PASS != IISPH_RHO && PASS != IISPH_DIJPJ) rhoi = a.rho_c[gi];
        if (PASS == IISPH_ADV) ui[0] = a.u[gi], ui[1] = a.v[gi], ui[2] = a.w[gi];
        if (PASS == IISPH_AII) ui[0] = a.uadv[gi], ui[1] = a.vadv[gi], ui[2] = a.wadv[gi];
        if (PASS == IISPH_AII) di[0] = a.dii0[gi], di[1] = a.dii1[gi], di[2] = a.dii2[gi];
        if (PASS == IISPH_SOLVE) dpi[0] = a.dijpj0[gi], dpi[1] = a.dijpj1[gi], dpi[2] = a.dijpj2[gi];
        if (PASS == IISPH_SOLVE) pi = a.piter[gi];
        if (PASS == IISPH_FORCE) pi = a.p[gi];
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *nxt = list_slot(a.lst, a.capg, s);
    struct Rec { ShiftRec P; uint32_t key, g; int t; };
    const auto load = [&](const uint32_t e, Rec &r) {
        const uint32_t j = LIST_J(e);
        r.P = a.P[j];
        r.key = a.skey[j];
        r.t = a.stype[j];
        r.g = a.perm[j];
    };
    const double dt = iisph_dt(a);
    const double rhoi1 = 1.0 / rhoi;
    // sums: s0 the scalar, v[3] the vector of the pass
    double s0 = 0.0, v[3] = {0.0, 0.0, 0.0}, av[3] = {0.0, 0.0, 0.0};
    unsigned npairs = 0;
    list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
        if (!live) return;
        const int tj = r.t & 7;
        const bool fluid = (a.fluid_mask >> tj) & 1u, solid = (a.solid_mask >> tj) & 1u;
        if (PASS == IISPH_V ? tj != (ti & 7) : (PASS == IISPH_DIJPJ ? !fluid : !(fluid || solid))) return;
        double xij[3];
        const double r2 = shift_dist(a, e, Pi, r.P, ci, r.key, xij);
        if (!shift_accept(a, r2, Pi.w, r.P.w)) return;
        npairs++;
        double wij, dw[3];
        const double hij = (Pi.w + r.P.w) * 0.5;
        shift_kernel<K, DIM>(a, xij, sqrt(r2), hij, wij, dw);
        const uint32_t gj = r.g;
        if constexpr (PASS == IISPH_V) {
            s0 += wij;                                                        // :41-42
        } else if constexpr (PASS == IISPH_RHO) {
            s0 += fluid ? a.m[gj] * wij : a.rho0 / a.V[gj] * wij;             // :49-50, :58-59
        } else if constexpr (PASS == IISPH_ADV) {
            const double vij[3] = {ui[0] - a.u[gj], ui[1] - a.v[gj], ui[2] - a.w[gj]};
            const double dwx = dw[0] * xij[0] + dw[1] * xij[1] + dw[2] * xij[2];
            const double eps = 0.01 * hij * hij;
            double fd, fv = 0.0;
            if (fluid) {
                fd = -a.m[gj] * rhoi1 * rhoi1;                                 // :140-146
                if (a.nu > 0.0) {                                              // :106-112
                    const double rhoij1 = 1.0 / (0.5 * (rhoi + a.rho_c[gj]));
                    fv = 2.0 * a.nu * a.m[gj] * rhoij1 * dwx / (r2 + eps);
                }
            } else {
                fd = -rhoi1 * rhoi1 * a.rho0 / a.V[gj];                        // :154-160
                if (a.nu > 0.0) {                                              // :123-131
                    const double phi_b = a.rho0 / (a.V[gj] * rhoi);
                    fv = 2.0 * a.nu * phi_b * dwx / (r2 + eps);
                }
            }
#pragma unroll
            for (int d = 0; d < 3; d++) {
                v[d] += fd * dw[d];
                av[d] += fv * vij[d];
            }
        } else if constexpr (PASS == IISPH_AII) {
            const double fac = mi * rhoi1 * rhoi1;
            const double dd = (di[0] - fac * dw[0]) * dw[0] + (di[1] - fac * dw[1]) * dw[1] + (di[2] - fac * dw[2]) * dw[2];
            if (fluid) {                                                       // :169-176, :198-207
                const double vd = (ui[0] - a.uadv[gj]) * dw[0] + (ui[1] - a.vadv[gj]) * dw[1] + (ui[2] - a.wadv[gj]) * dw[2];
                s0 += dt * a.m[gj] * vd;
                v[0] += a.m[gj] * dd;
            } else {                                                           // :184-191, :217-225
                const double phi_b = a.rho0 / a.V[gj];
                const double vd = (ui[0] - a.u[gj]) * dw[0] + (ui[1] - a.v[gj]) * dw[1] + (ui[2] - a.w[gj]) * dw[2];
                s0 += dt * phi_b * vd;
                v[0] += phi_b * dd;
            }
        } else if constexpr (PASS == IISPH_DIJPJ) {                            // :234-240
            const double rj1 = 1.0 / a.rho_c[gj];
            const double fac = -a.m[gj] * rj1 * rj1 * a.piter[gj];
#pragma unroll
            for (int d = 0; d < 3; d++) v[d] += fac * dw[d];
        } else if constexpr (PASS == IISPH_SOLVE) {
            if (fluid) {                                                       // :278-296
                const double fac = mi * rhoi1 * rhoi1 * pi;
                const double pj = a.piter[gj];
                const double t0 = dpi[0] - a.dii0[gj] * pj - (a.dijpj0[gj] - fac * dw[0]);
                const double t1 = dpi[1] - a.dii1[gj] * pj - (a.dijpj1[gj] - fac * dw[1]);
                const double t2 = dpi[2] - a.dii2[gj] * pj - (a.dijpj2[gj] - fac * dw[2]);
                s0 += a.m[gj] * (t0 * dw[0] + t1 * dw[1] + t2 * dw[2]);
            } else {                                                           // :349-355
                s0 += a.rho0 / a.V[gj] * (dpi[0] * dw[0] + dpi[1] * dw[1] + dpi[2] * dw[2]);
            }
        } else {                                                               // IISPH_FORCE
            double fac;
            if (fluid) {                                                       // :373-380
                const double rj1 = 1.0 / a.rho_c[gj];
                fac = -a.m[gj] * (pi * rhoi1 * rhoi1 + a.p[gj] * rj1 * rj1);
            } else {                                                           // :397-402
                fac = -pi * rhoi1 * rhoi1 * a.rho0 / a.V[gj];
            }
#pragma unroll
            for (int d = 0; d < 3; d++) v[d] += fac * dw[d];
        }
    });
    pairs_flush(a, npairs);
    if (!active) return;
    const uint32_t g = gi;
    if constexpr (PASS == IISPH_V) {
        a.V[g] = s0;
    } else if constexpr (PASS == IISPH_RHO) {
        a.rho[g] = s0;
    } else if constexpr (PASS == IISPH_ADV) {
        a.dii0[g] = v[0]; a.dii1[g] = v[1]; a.dii2[g] = v[2];
        a.uadv[g] = ui[0] + dt * (a.gx + av[0]);                               // :94-98
        a.vadv[g] = ui[1] + dt * (a.gy + av[1]);
        a.wadv[g] = ui[2] + dt * (a.gz + av[2]);
    } else if constexpr (PASS == IISPH_AII) {
        a.rho_adv[g] = rhoi + s0;                                              // :164-167
        a.aii[g] = v[0];
        const double p = a.p[g];
        a.p0[g] = p;
        a.piter[g] = 0.5 * p;
    } else if constexpr (PASS == IISPH_DIJPJ) {
        a.dijpj0[g] = v[0]; a.dijpj1[g] = v[1]; a.dijpj2[g] = v[2];
    } else if constexpr (PASS == IISPH_SOLVE) {                                // post_loop :298-318
        const double dt2 = dt * dt;
        const double tmp = a.rho0 - a.rho_adv[g] - s0 * dt2;
        const double dnr = a.aii[g] * dt2;
        double p = 0.0;
        if (fabs(dnr) > 1e-9) p = fmax((1.0 - a.omega) * pi + a.omega / dnr * tmp, 0.0);
        a.comp[g] = p != 0.0 ? fabs(p * dnr - tmp) + a.rho0 : a.rho0;
        a.pnext[g] = p;
    } else {                                                                   // post_loop :382-389
        a.au[g] = (float)v[0]; a.av[g] = (float)v[1]; a.aw[g] = (float)v[2];
        const double ua = a.uadv[g], va = a.vadv[g], wa = a.wadv[g];
        a.dt_cfl[g] = (float)(2.0 * sqrt(ua * ua + va * va + wa * wa));
        a.dt_force[g] = (float)(2.0 * (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
    }
}

// the end of PressureSolve's post-loop for the pool range [off, off + n) of one array:
// piter = p = the new pressure
__global__ void k_iisph_commit(const IisphArgs a, const long long off, const long long n)
{
    if (*(volatile const int *)&a.st->done) return;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double p = a.pnext[off + i];
    a.piter[off + i] = p;
    a.p[off + i] = p;
}

// PressureSolve.reduce (:320-328) of one fluid, part 1: each block sums (compression > 0) and
// compression over its IISPH_RED particles of [off, off + n) in a fixed tree order
__global__ void __launch_bounds__(IISPH_RED) k_iisph_partials(const IisphArgs a, const long long off, const long long n)
{
    if (*(volatile const int *)&a.st->done) return;
    __shared__ double sc[IISPH_RED], sv[IISPH_RED];
    const long long i = (long long)blockIdx.x * IISPH_RED + threadIdx.x;
    double c = 0.0, v = 0.0;
    if (i < n) {
        v = a.comp[off + i];
        c = v > 0.0 ? 1.0 : 0.0;
    }
    sc[threadIdx.x] = c;
    sv[threadIdx.x] = v;
    __syncthreads();
    for (int o = IISPH_RED / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            sc[threadIdx.x] += sc[threadIdx.x + o];
            sv[threadIdx.x] += sv[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        a.part[2 * blockIdx.x] = sc[0];
        a.part[2 * blockIdx.x + 1] = sv[0];
    }
}

// part 2, one block: the partials of fluid `arr` in a fixed order -> the compression of that
// fluid; `last`: the last fluid of the iteration, which then counts it and decides
__global__ void __launch_bounds__(IISPH_RED) k_iisph_converge(const IisphArgs a, const long long nb, const int arr, const int last)
{
    if (*(volatile const int *)&a.st->done) return;
    __shared__ double sc[IISPH_RED], sv[IISPH_RED];
    double c = 0.0, v = 0.0;
    for (long long b = threadIdx.x; b < nb; b += IISPH_RED) {
        c += a.part[2 * b];
        v += a.part[2 * b + 1];
    }
    sc[threadIdx.x] = c;
    sv[threadIdx.x] = v;
    __syncthreads();
    for (int o = IISPH_RED / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            sc[threadIdx.x] += sc[threadIdx.x + o];
            sv[threadIdx.x] += sv[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const double avg = sc[0] > 0.0 ? sv[0] / sc[0] : a.rho0;
    a.st->comp[arr] = fabs(avg - a.rho0) / a.rho0;
    if (!last) return;
    const int it = a.st->it + 1;
    a.st->it = it;
    bool conv = true;   // PressureSolve.converged (:330-341) of every fluid
    for (int f = 0; f < B200SPH_MAX_ARRAYS; f++)
        if (((a.fluid_mask >> f) & 1u) && a.st->comp[f] > a.tol) conv = false;
    if (it >= a.min_it && (conv || it == a.max_it)) a.st->done = 1;
}

// IISPHStep.stage1 (:22-34): u = uadv + dt au, x += dt u, on the real particles of array `arr`
// (-1: every array whose bit is in mask)
struct StageIisphArgs {
    double *x, *y, *z, *u, *v, *w;
    const double *uadv, *vadv, *wadv;
    const float *au, *av, *aw;
    const uint8_t *ptype;
    long long pool_end;
    unsigned mask;
    double dt;
    const double *tc;
};
__global__ void k_stage_iisph(const StageIisphArgs a)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    const uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST) || !((a.mask >> (t & 7)) & 1u)) return;
    const double dt = a.tc ? a.tc[0] : a.dt;
    const double u = a.uadv[g] + dt * (double)a.au[g];
    const double v = a.vadv[g] + dt * (double)a.av[g];
    const double w = a.wadv[g] + dt * (double)a.aw[g];
    a.u[g] = u; a.v[g] = v; a.w[g] = w;
    a.x[g] += dt * u;
    a.y[g] += dt * v;
    a.z[g] += dt * w;
}
