// crksph_kernels.cuh -- conservative reproducing-kernel SPH: the two evaluations of
// CRKSPHScheme.get_equations (pysph/sph/wc/crksph.py:978-1127) over the persistent neighbour
// lists, and CRKSPHStep.  Part of the single translation unit b200sph.cu (included there, in this
// order; not a stand-alone header).
//
// One THREAD per destination walks its list (list_walk) and keeps the sources of the fluid array;
// the geometry is the particle shifting's (shift_dist, shift_accept, shift_kernel): x_ij, r^2 and
// the accept test in fp64, a periodic image from the entry's cell offset, the kernel polynomial in
// fp32 and every sum in fp64.  Every property is fp64.  A pass boundary lies wherever a body reads
// a source value an earlier Group of the same evaluation writes:
//   evaluation 0
//     CRK_VOL    StateEquation + SpeedOfSound (:786-810) as the prologue, NumberDensity (:391-406):
//                p, cs, V = sum_j W(x_ij, h_i)
//     CRK_PRE    CRKSPHPreStep (:32-167): the moments m0, m1, m2 and their gradients with
//                h_ij and V_j = 1 / V_j, m2 inverted by gj_solve with d right-hand sides:
//                ai, bi, gradai, gradbi
//     CRK_RHO    CRKSPHSymmetric's cwij + SummationDensityCRKSPH (:409-441), with the second
//                StateEquation + SpeedOfSound folded into its post-loop: rho, p, cs
//     CRK_GRADV  CRKSPHSymmetric's destination-side gradient DWI + VelocityGradient (:444-477): gradv
//     CRK_MOM    CRKSPHSymmetric + MomentumEquation (:480-632) + LaminarViscosity (wc/viscosity.py,
//                nu != 0), which reads the corrected, symmetrised DWIJ: au, av, aw
//   evaluation 1
//     CRK_ENERGY CRKSPHSymmetric + EnergyEquation (:635-783): ae
// The limiter's min / max are Python's builtins (crk_min, crk_max): min(a, b) is a unless b < a,
// so min(1, nan) is 1 where gradv vanishes (r_ij = 0 / 0).
// --------------------------------------------------------------------------
#define CRK_NT 128

enum { CRK_VOL = 0, CRK_PRE, CRK_RHO, CRK_GRADV, CRK_MOM, CRK_ENERGY };

struct CrkArgs {
    ShiftRec *P;                      // [n] (x, y, z, h) by sorted slot (k_crksph_pack)
    const uint32_t *perm, *cnt, *lst, *skey;
    const uint8_t *stype;
    const double *h, *m, *u, *v, *w, *u0, *v0, *w0, *e;
    double *rho, *p, *cs, *V, *ai, *au, *av, *aw, *ae;
    double *bi[3], *gai[3];           // B_i^a, dA_i / dx_g
    double *gbi[9], *gv[9];           // dB_i^a / dx_g at [3 g + a]; dv^a / dx^b at [3 a + b]
    unsigned long long *pair_counter;
    long long n;
    int capg;
    int ncx, ncy, zorder;
    int per[3];
    double L[3];
    double kr, kfac;
    unsigned fluid_mask;
    double gamma, gx, gy, gz;
    double cl, cq, eta_crit, eta_fold;        // MomentumEquation
    double cl_e, cq_e, eta_crit_e, eta_fold_e; // EnergyEquation
    double nu, eta;                            // LaminarViscosity (nu 0: absent)
};

// Python's min / max of two numbers: the first unless the second compares below (above) it
__device__ __forceinline__ double crk_min(const double a, const double b) { return b < a ? b : a; }
__device__ __forceinline__ double crk_max(const double a, const double b) { return b > a ? b : a; }

// index of (a, b), a <= b, in the packed upper triangle of a symmetric DIM x DIM matrix
template <int DIM> __device__ __forceinline__ constexpr int crk_sym(const int a, const int b)
{
    return a <= b ? a * DIM - a * (a - 1) / 2 + (b - a) : b * DIM - b * (b - 1) / 2 + (a - b);
}

__global__ void k_crksph_pack(const CrkArgs a, const double *x, const double *y, const double *z)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const uint32_t g = a.perm[s];
    a.P[s] = ShiftRec{x[g], y[g], z[g], a.h[g]};
}

// One side of CRKSPHSymmetric (:354-388): the corrected gradient of particle k with its own
// smoothing length, sg = +1 for the destination (temp), -1 for the source (temp1; B and grad B
// enter with x_ji = -x_ij and A with -dW)
template <int K, int DIM>
__device__ __forceinline__ void crk_side(const CrkArgs &a, const uint32_t k, const double sg, const double xij[3],
                                         const double rij, const double hk, double &bx, double dw[3])
{
    double wk, dwk[3];
    shift_kernel<K, DIM>(a, xij, rij, hk, wk, dwk);
    const double ak = a.ai[k];
    bx = 0.0;
#pragma unroll
    for (int al = 0; al < DIM; al++) bx = sg > 0.0 ? bx + a.bi[al][k] * xij[al] : bx - a.bi[al][k] * xij[al];
#pragma unroll
    for (int g = 0; g < DIM; g++) {
        double dbx = 0.0;
#pragma unroll
        for (int al = 0; al < DIM; al++) dbx = sg > 0.0 ? dbx + a.gbi[3 * g + al][k] * xij[al] : dbx - a.gbi[3 * g + al][k] * xij[al];
        double t = ((sg * ak) * dwk[g] + a.gai[g][k] * wk) * (1 + bx);
        t += ak * (dbx + a.bi[g][k]) * wk;
        dw[g] = t;
    }
}

// the limiter and the artificial pressures of MomentumEquation / EnergyEquation (:588-627,
// :715-754); vi, vj: the velocities the body differences (u for momentum, u0 for energy).  Returns
// (p_i + p_j + Q_i + Q_j)
template <int DIM>
__device__ __forceinline__ double crk_q(const CrkArgs &a, const uint32_t gi, const uint32_t gj, const double xij[3],
                                        const double vi[3], const double vj[3], const double hi, const double hj,
                                        const double hij, const double cl, const double cq, const double eta_crit,
                                        const double eta_fold)
{
    double tmpri = 0.0, tmprj = 0.0;
#pragma unroll
    for (int al = 0; al < DIM; al++)
#pragma unroll
        for (int be = 0; be < DIM; be++) {
            tmpri += a.gv[3 * al + be][gi] * xij[al] * xij[be];
            tmprj += a.gv[3 * al + be][gj] * xij[al] * xij[be];
        }
    const double rij = tmpri / tmprj;
    const double tmprij = crk_min(1.0, 4 * rij / ((1 + rij) * (1 + rij)));
    double phiij = crk_max(0.0, tmprij);
    double tmpxij = 0.0;
#pragma unroll
    for (int al = 0; al < DIM; al++) tmpxij += xij[al] * xij[al];
    const double tmpxij2 = sqrt(tmpxij);
    const double etaij = crk_min(tmpxij2 / hi, tmpxij2 / hj);
    if (etaij < eta_crit) {
        const double tmpphi = (etaij - eta_crit) / eta_fold;
        phiij = phiij * exp(-tmpphi * tmpphi);
    }
    double uh[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int al = 0; al < DIM; al++) {
        double s = 0.0;
#pragma unroll
        for (int be = 0; be < DIM; be++) s += (a.gv[3 * al + be][gi] + a.gv[3 * al + be][gj]) * xij[be];
        uh[al] = vi[al] - vj[al] - 0.5 * phiij * s;
    }
    double ux = 0.0;
#pragma unroll
    for (int al = 0; al < DIM; al++) ux += uh[al] * xij[al];
    const double eps = 0.01 * hij * hij;
    // (the reference divides by tmpxij / h_i in both: h_i where h_j would be expected)
    const double mui = crk_min(0.0, ux / (tmpxij / hi + eps * hi));
    const double muj = crk_min(0.0, ux / (tmpxij / hi + eps * hj));
    const double qi = a.rho[gi] * (-cl * a.cs[gi] * mui + cq * mui * mui);
    const double qj = a.rho[gj] * (-cl * a.cs[gj] * muj + cq * muj * muj);
    return a.p[gi] + a.p[gj] + qi + qj;
}

template <int K, int DIM, int PASS>
__global__ void __launch_bounds__(CRK_NT) k_crksph(const CrkArgs a)
{
    constexpr int NS = DIM * (DIM + 1) / 2;   // a packed symmetric DIM x DIM matrix
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * CRK_NT + threadIdx.x;
    int ti = 0, count = 0;
    bool active = false;
    if (s < a.n) {
        ti = a.stype[s];
        active = ((a.fluid_mask >> (ti & 7)) & 1u) && !(ti & PT_GHOST);
    }
    ShiftRec Pi = {0.0, 0.0, 0.0, 0.0};
    uint32_t ci[3] = {0u, 0u, 0u}, gi = 0;
    double ui[3] = {0.0, 0.0, 0.0}, ai = 0.0, bi[3] = {0.0, 0.0, 0.0};
    if (active) {
        Pi = a.P[s];
        count = (int)a.cnt[s];
        grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, a.skey[s], ci[0], ci[1], ci[2]);
        gi = a.perm[s];
        if (PASS == CRK_VOL) {                                                     // :800-810
            const double rho = a.rho[gi];
            const double p = (a.gamma - 1) * rho * a.e[gi];
            a.p[gi] = p;
            a.cs[gi] = sqrt(a.gamma * p / rho);
        }
        if (PASS == CRK_GRADV || PASS == CRK_MOM) ui[0] = a.u[gi], ui[1] = a.v[gi], ui[2] = a.w[gi];
        if (PASS == CRK_ENERGY) ui[0] = a.u0[gi], ui[1] = a.v0[gi], ui[2] = a.w0[gi];
        if (PASS == CRK_RHO) {
            ai = a.ai[gi];
#pragma unroll
            for (int al = 0; al < DIM; al++) bi[al] = a.bi[al][gi];
        }
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
    // the pass's sums: s0, s1 scalars, v[3] a vector, gm[9] a DIM x DIM matrix; CRK_PRE's moments
    double s0 = 0.0, s1 = 0.0, v[3] = {0.0, 0.0, 0.0}, gm[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    double m0 = 0.0, m1[DIM], m2[NS], gm0[DIM], gm1[DIM * DIM], gm2[DIM * NS];
#pragma unroll
    for (int k = 0; k < DIM; k++) m1[k] = gm0[k] = 0.0;
#pragma unroll
    for (int k = 0; k < NS; k++) m2[k] = 0.0;
#pragma unroll
    for (int k = 0; k < DIM * DIM; k++) gm1[k] = 0.0;
#pragma unroll
    for (int k = 0; k < DIM * NS; k++) gm2[k] = 0.0;
    unsigned npairs = 0;
    list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
        if (!live || !((a.fluid_mask >> (r.t & 7)) & 1u)) return;
        double xij[3];
        const double r2 = shift_dist(a, e, Pi, r.P, ci, r.key, xij);
        if (!shift_accept(a, r2, Pi.w, r.P.w)) return;
        npairs++;
        const uint32_t gj = r.g;
        const double rij = sqrt(r2);
        const double hij = (Pi.w + r.P.w) * 0.5;
        if constexpr (PASS == CRK_VOL) {                                           // :405-406
            double wi, dwi[3];
            shift_kernel<K, DIM>(a, xij, rij, Pi.w, wi, dwi);
            s0 += wi;
        } else if constexpr (PASS == CRK_PRE) {                                    // :83-109
            double wij, dw[3];
            shift_kernel<K, DIM>(a, xij, rij, hij, wij, dw);
            const double Vj = 1.0 / a.V[gj];
            m0 += Vj * wij;
#pragma unroll
            for (int al = 0; al < DIM; al++) {
                m1[al] += Vj * wij * xij[al];
#pragma unroll
                for (int be = al; be < DIM; be++) m2[crk_sym<DIM>(al, be)] += Vj * wij * xij[al] * xij[be];
            }
#pragma unroll
            for (int g = 0; g < DIM; g++) {
                gm0[g] += Vj * dw[g];
#pragma unroll
                for (int al = 0; al < DIM; al++) {
                    gm1[DIM * g + al] += Vj * (xij[al] * dw[g] + (al == g ? wij : 0.0));
#pragma unroll
                    for (int be = al; be < DIM; be++) {
                        const double t = (be == g ? xij[al] : 0.0) + (al == g ? xij[be] : 0.0);
                        gm2[NS * g + crk_sym<DIM>(al, be)] += Vj * (xij[al] * xij[be] * dw[g] + t * wij);
                    }
                }
            }
        } else if constexpr (PASS == CRK_RHO) {                                    // :362-375, :434-438
            double wij, dw[3];
            shift_kernel<K, DIM>(a, xij, rij, hij, wij, dw);
            double bx = 0.0;
#pragma unroll
            for (int al = 0; al < DIM; al++) bx += bi[al] * xij[al];
            const double Vj = 1.0 / a.V[gj];
            const double fac = Vj * (ai * (1 + bx)) * wij;
            s0 += a.m[gi] * fac;
            s1 += Vj * fac;
        } else if constexpr (PASS == CRK_GRADV) {                                  // :473-477
            double bx, dwi[3];
            crk_side<K, DIM>(a, gi, 1.0, xij, rij, Pi.w, bx, dwi);
            const double Vj = 1.0 / a.V[gj];
            const double vij[3] = {ui[0] - a.u[gj], ui[1] - a.v[gj], ui[2] - a.w[gj]};
#pragma unroll
            for (int al = 0; al < DIM; al++)
#pragma unroll
                for (int be = 0; be < DIM; be++) gm[DIM * al + be] += -Vj * vij[al] * dwi[be];
        } else {                                                                   // CRK_MOM, CRK_ENERGY
            double wij, dwij[3], bxi, bxj, dwi[3], dwj[3];
            shift_kernel<K, DIM>(a, xij, rij, hij, wij, dwij);
            crk_side<K, DIM>(a, gi, 1.0, xij, rij, Pi.w, bxi, dwi);
            crk_side<K, DIM>(a, gj, -1.0, xij, rij, r.P.w, bxj, dwj);
#pragma unroll
            for (int g = 0; g < DIM; g++) dwij[g] = 0.5 * (dwi[g] - dwj[g]);       // :386
            const double Vi = 1.0 / a.V[gi], Vj = 1.0 / a.V[gj];
            if constexpr (PASS == CRK_MOM) {
                const double vj[3] = {a.u[gj], a.v[gj], a.w[gj]};
                const double pq = crk_q<DIM>(a, gi, gj, xij, ui, vj, Pi.w, r.P.w, hij, a.cl, a.cq, a.eta_crit, a.eta_fold);
                const double fac = -(1.0 / a.m[gi]) * Vi * Vj * pq;                // :629-632
#pragma unroll
                for (int d = 0; d < 3; d++) v[d] += fac * dwij[d];
                if (a.nu != 0.0) {                                                 // viscosity.py:12-27
                    const double rhoa = a.rho[gi], rhob = a.rho[gj];
                    const double fij = dwij[0] * xij[0] + dwij[1] * xij[1] + dwij[2] * xij[2];
                    const double tmp = a.m[gj] * 4 * a.nu * fij / ((rhoa + rhob) * (r2 + a.eta * hij * hij));
                    v[0] += tmp * (ui[0] - vj[0]);
                    v[1] += tmp * (ui[1] - vj[1]);
                    v[2] += tmp * (ui[2] - vj[2]);
                }
            } else {                                                               // :756-783
                const double u0j[3] = {a.u0[gj], a.v0[gj], a.w0[gj]};
                const double pq = crk_q<DIM>(a, gi, gj, xij, ui, u0j, Pi.w, r.P.w, hij, a.cl_e, a.cq_e, a.eta_crit_e,
                                             a.eta_fold_e);
                const double fac = -(1.0 / a.m[gi]) * Vi * Vj * pq;
                const double uj[3] = {a.u[gj], a.v[gj], a.w[gj]}, uii[3] = {a.u[gi], a.v[gi], a.w[gi]};
                double aeij = 0.0;
#pragma unroll
                for (int d = 0; d < DIM; d++) aeij += (u0j[d] + uj[d] - ui[d] - uii[d]) * (fac * dwij[d]);
                const double si = a.p[gi] / pow(a.rho[gi], a.gamma);
                const double sj = a.p[gj] / pow(a.rho[gj], a.gamma);
                const double smin = crk_min(fabs(si), fabs(sj)), smax = crk_max(fabs(si), fabs(sj));
                double fij = 0.5;
                const double sdiff = si - sj;
                if (sdiff * aeij > 0) fij = smin / (smin + smax);
                else if (sdiff * aeij < 0) fij = smax / (smin + smax);
                s0 += 0.5 * fij * aeij;
            }
        }
    });
    pairs_flush(a, npairs);
    if (!active) return;
    const uint32_t g = gi;
    if constexpr (PASS == CRK_VOL) {
        a.V[g] = s0;
    } else if constexpr (PASS == CRK_PRE) {                                        // :111-167
        double aug[DIM][2 * DIM], m2inv[DIM][DIM];
#pragma unroll
        for (int i = 0; i < DIM; i++)
#pragma unroll
            for (int j = 0; j < DIM; j++) {
                aug[i][j] = m2[crk_sym<DIM>(i, j)];
                aug[i][DIM + j] = m2inv[i][j] = i == j ? 1.0 : 0.0;
            }
        const bool ok = gj_solve<DIM, DIM>(aug);
        double A = 1.0, B[3] = {0.0, 0.0, 0.0}, gA[3] = {0.0, 0.0, 0.0}, gB[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        if (ok && npairs >= 2) {
#pragma unroll
            for (int i = 0; i < DIM; i++)
#pragma unroll
                for (int j = 0; j < DIM; j++) m2inv[i][j] = aug[i][DIM + j];
            double tv[DIM];
#pragma unroll
            for (int i = 0; i < DIM; i++) {
                double t = 0.0;
#pragma unroll
                for (int j = 0; j < DIM; j++) t += m2inv[i][j] * m1[j];
                tv[i] = t;
            }
            double dt = 0.0;
#pragma unroll
            for (int i = 0; i < DIM; i++) dt += tv[i] * m1[i];
            A = 1.0 / (m0 - dt);
#pragma unroll
            for (int i = 0; i < DIM; i++) B[i] = -tv[i];
#pragma unroll
            for (int gg = 0; gg < DIM; gg++) {
                double t1 = gm0[gg];
#pragma unroll
                for (int al = 0; al < DIM; al++) {
                    double t2 = 0.0;
#pragma unroll
                    for (int be = 0; be < DIM; be++) {
                        t1 -= m2inv[al][be] * (m1[be] * gm1[DIM * gg + al] + m1[al] * gm1[DIM * gg + be]);
                        t2 -= m2inv[al][be] * gm1[DIM * gg + be];
#pragma unroll
                        for (int ph = 0; ph < DIM; ph++)
#pragma unroll
                            for (int ps = 0; ps < DIM; ps++) {
                                const double q = m2inv[al][ph] * m2inv[ps][be] * gm2[NS * gg + crk_sym<DIM>(ph, ps)];
                                t1 += q * m1[be] * m1[al];
                                t2 += q * m1[be];
                            }
                    }
                    gB[3 * gg + al] = t2;
                }
                gA[gg] = -A * A * t1;
            }
        }
        a.ai[g] = A;
#pragma unroll
        for (int i = 0; i < DIM; i++) {
            a.bi[i][g] = B[i];
            a.gai[i][g] = gA[i];
#pragma unroll
            for (int j = 0; j < DIM; j++) a.gbi[3 * i + j][g] = gB[3 * i + j];
        }
    } else if constexpr (PASS == CRK_RHO) {                                        // :440-441, :800-810
        const double rho = s0 / s1;
        a.rho[g] = rho;
        const double p = (a.gamma - 1) * rho * a.e[g];
        a.p[g] = p;
        a.cs[g] = sqrt(a.gamma * p / rho);
    } else if constexpr (PASS == CRK_GRADV) {
#pragma unroll
        for (int al = 0; al < DIM; al++)
#pragma unroll
            for (int be = 0; be < DIM; be++) a.gv[3 * al + be][g] = gm[DIM * al + be];
    } else if constexpr (PASS == CRK_MOM) {                                        // :553-556
        a.au[g] = a.gx + v[0];
        a.av[g] = a.gy + v[1];
        a.aw[g] = a.gz + v[2];
    } else {
        a.ae[g] = s0;
    }
}

// CRKSPHStep (crksph.py:884-900) on the real particles of array `arr` (-1: every array):
//   1: u0 = u    2: u += dt au    3: e += dt ae, x += dt / 2 (u + u0)
struct StageCrkArgs {
    double *x, *y, *z, *u, *v, *w, *u0, *v0, *w0, *e;
    const double *au, *av, *aw, *ae;
    const uint8_t *ptype;
    long long pool_end;
    unsigned mask;
    int which;
    double dt;
    const double *tc;
};
__global__ void k_stage_crksph(const StageCrkArgs a)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    const uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST) || !((a.mask >> (t & 7)) & 1u)) return;
    const double dt = a.tc ? a.tc[0] : a.dt;
    if (a.which == 1) {
        a.u0[g] = a.u[g];
        a.v0[g] = a.v[g];
        a.w0[g] = a.w[g];
    } else if (a.which == 2) {
        a.u[g] += a.au[g] * dt;
        a.v[g] += a.av[g] * dt;
        a.w[g] += a.aw[g] * dt;
    } else {
        a.e[g] += a.ae[g] * dt;
        a.x[g] += 0.5 * dt * (a.u[g] + a.u0[g]);
        a.y[g] += 0.5 * dt * (a.v[g] + a.v0[g]);
        a.z[g] += 0.5 * dt * (a.w[g] + a.w0[g]);
    }
}
