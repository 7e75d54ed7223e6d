// gtvf_kernels.cuh -- the generalised transport-velocity formulation: the two evaluations of
// GTVFScheme.get_equations (pysph/sph/wc/gtvf.py:586-662) over the persistent neighbour lists,
// and GTVFStep.  Part of the single translation unit b200sph.cu (included there, in this order;
// not a stand-alone header).
//
// One THREAD per destination walks its list (list_walk) and keeps the sources of the arrays the
// pass reads; the geometry is the particle shifting's (shift_dist, shift_accept, shift_kernel):
// x_ij, r^2 and the accept test in fp64, a periodic image from the entry's cell offset, the kernel
// polynomial in fp32 and every sum in fp64.  A pass boundary lies wherever a body reads a source
// value an earlier Group of the same evaluation writes:
//   evaluation 0
//     GTVF_WALLV  SetWallVelocity (transport_velocity.py:84-134), every wall over the fluids:
//                 wij, uf, ug
//     GTVF_CONT   ContinuityEquationGTVF (gtvf.py:101-121) over the fluids and ContinuitySolid
//                 (transport_velocity.py:157-173) over the walls: arho
//   evaluation 1
//     GTVF_RHO    CorrectDensity (gtvf.py:124-148) over every array, StateEquation
//                 (transport_velocity.py:176-216, b = 1) folded into its post-loop: rho, rhodiv,
//                 p.  CorrectDensity.initialize's rho0 = rho is made before the pass (the host
//                 copies it), so the pass reads rho0 only
//     GTVF_WALLP  VolumeSummation (transport_velocity.py:61-75) over every array and the
//                 transport-velocity SolidWallPressureBC (:641-736, b = 1) over the fluids: V, p,
//                 wij, and the wall's rho = rho0 (p / pref + 1)
//     GTVF_MOM    MomentumEquationPressureGradient (gtvf.py:151-250; auhat with the gradient at
//                 0.5 h_ij of the same x_ij), MomentumEquationArtificialViscosity
//                 (transport_velocity.py:389-448, alpha > 0), MomentumEquationViscosity
//                 (gtvf.py:253-288, nu > 0) over every array, MomentumEquationArtificialStress
//                 (gtvf.py:291-348) over the fluids: au, auhat, p0
// --------------------------------------------------------------------------
#define GTVF_NT 128

enum { GTVF_WALLV = 0, GTVF_CONT, GTVF_RHO, GTVF_WALLP, GTVF_MOM };

struct GtvfArgs {
    ShiftRec *P;                      // [n] (x, y, z, h) by sorted slot (k_gtvf_pack)
    const uint32_t *perm, *cnt, *lst, *skey;
    const uint8_t *stype;
    const double *x, *y, *z, *h, *m, *u, *v, *w, *uh, *vh, *wh, *rho0;
    double *rho, *pf, *rhodiv, *p0, *ug, *vg, *wg;
    float *p, *arho, *au, *av, *aw, *auh, *avh, *awh, *vol, *wij, *uf, *vf, *wf;
    unsigned long long *pair_counter;
    long long n;
    int capg;
    int ncx, ncy, zorder;
    int per[3];
    double L[3];
    double kr, kfac;
    unsigned fluid_mask, solid_mask;
    double rho0c, pref, c0, alpha, nu, gx, gy, gz;
};

__global__ void k_gtvf_pack(const GtvfArgs a)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n) return;
    const uint32_t g = a.perm[s];
    a.P[s] = ShiftRec{a.x[g], a.y[g], a.z[g], a.h[g]};
}

template <int K, int DIM, int PASS>
__global__ void __launch_bounds__(GTVF_NT) k_gtvf(const GtvfArgs a)
{
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * GTVF_NT + threadIdx.x;
    constexpr bool WALL = PASS == GTVF_WALLV || PASS == GTVF_WALLP;
    int ti = 0, count = 0;
    bool active = false;
    if (s < a.n) {
        ti = a.stype[s];
        active = (((WALL ? a.solid_mask : a.fluid_mask) >> (ti & 7)) & 1u) && !(ti & PT_GHOST);
    }
    ShiftRec Pi = {0.0, 0.0, 0.0, 0.0};
    uint32_t ci[3] = {0u, 0u, 0u}, gi = 0;
    double rhoi = 1.0, pi = 0.0, p0i = 0.0, ui[3] = {0.0, 0.0, 0.0}, uhi[3] = {0.0, 0.0, 0.0}, gw[3] = {0.0, 0.0, 0.0};
    if (active) {
        Pi = a.P[s];
        count = (int)a.cnt[s];
        grid_decode(a.zorder, (uint32_t)a.ncx, (uint32_t)a.ncy, a.skey[s], ci[0], ci[1], ci[2]);
        gi = a.perm[s];
        if (PASS == GTVF_CONT || PASS == GTVF_MOM) rhoi = a.rho[gi];
        if (PASS != GTVF_RHO && PASS != GTVF_WALLV) ui[0] = a.u[gi], ui[1] = a.v[gi], ui[2] = a.w[gi];
        if (PASS == GTVF_CONT || PASS == GTVF_MOM) uhi[0] = a.uh[gi], uhi[1] = a.vh[gi], uhi[2] = a.wh[gi];
        if (PASS == GTVF_MOM) {
            pi = a.pf[gi];
            p0i = fmin(10.0 * fabs(pi), a.pref);                                    // gtvf.py:227
        }
        if (PASS == GTVF_WALLP) {                                                  // (g - a_wall), tv:721-723
            gw[0] = a.gx - (double)a.au[gi];
            gw[1] = a.gy - (double)a.av[gi];
            gw[2] = a.gz - (double)a.aw[gi];
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
    // the pass's sums: s0, s1 scalars, v[3], vh[3] vectors
    double s0 = 0.0, s1 = 0.0, v[3] = {0.0, 0.0, 0.0}, vh[3] = {0.0, 0.0, 0.0};
    unsigned npairs = 0;
    list_walk<Rec>(nxt, count, cmax, load, [&](const bool live, const uint32_t e, const Rec &r) {
        if (!live) return;
        const int tj = r.t & 7;
        const bool fluid = (a.fluid_mask >> tj) & 1u, solid = (a.solid_mask >> tj) & 1u;
        // SetWallVelocity, SolidWallPressureBC and the artificial stress take the fluids only
        if (PASS == GTVF_WALLV ? !fluid : !(fluid || solid)) return;
        double xij[3];
        const double r2 = shift_dist(a, e, Pi, r.P, ci, r.key, xij);
        if (!shift_accept(a, r2, Pi.w, r.P.w)) return;
        npairs++;
        double wij, dw[3];
        const double hij = (Pi.w + r.P.w) * 0.5;
        const double rij = sqrt(r2);
        shift_kernel<K, DIM>(a, xij, rij, hij, wij, dw);
        const uint32_t gj = r.g;
        if constexpr (PASS == GTVF_WALLV) {                                        // tv:106-117
            s0 += wij;
            v[0] += a.u[gj] * wij;
            v[1] += a.v[gj] * wij;
            v[2] += a.w[gj] * wij;
        } else if constexpr (PASS == GTVF_CONT) {
            double vij[3];
            if (fluid) {                                                           // gtvf.py:113-121
                vij[0] = uhi[0] - a.uh[gj]; vij[1] = uhi[1] - a.vh[gj]; vij[2] = uhi[2] - a.wh[gj];
            } else {                                                               // tv:164-173
                vij[0] = ui[0] - a.ug[gj]; vij[1] = ui[1] - a.vg[gj]; vij[2] = ui[2] - a.wg[gj];
            }
            const double vd = dw[0] * vij[0] + dw[1] * vij[1] + dw[2] * vij[2];
            s0 += rhoi * a.m[gj] / a.rho[gj] * vd;
        } else if constexpr (PASS == GTVF_RHO) {                                   // gtvf.py:143-145
            const double mw = a.m[gj] * wij;
            s0 += mw;
            s1 += mw / a.rho0[gj];            // a wall with rho0 = 0 gives inf (or nan): min(1, .) = 1
        } else if constexpr (PASS == GTVF_WALLP) {
            s0 += wij;                                                             // VolumeSummation
            if (fluid) {                                                           // tv:715-728
                const double gdx = gw[0] * xij[0] + gw[1] * xij[1] + gw[2] * xij[2];
                s1 += a.pf[gj] * wij + a.rho[gj] * gdx * wij;
                v[0] += wij;
            }
        } else {                                                                   // GTVF_MOM
            const double rhoj = a.rho[gj], mj = a.m[gj];
            const double pj = fluid ? a.pf[gj] : (double)a.p[gj];
            const double rhoi2 = rhoi * rhoi;
            const double fp = -mj * (pi / rhoi2 + pj / (rhoj * rhoj));              // gtvf.py:232-241
            double dwh[3], wh;
            shift_kernel<K, DIM>(a, xij, rij, 0.5 * hij, wh, dwh);                 // gtvf.py:243-250
            const double fh = -p0i * mj / rhoi2;
            double uj[3] = {a.u[gj], a.v[gj], a.w[gj]};
            const double vij[3] = {ui[0] - uj[0], ui[1] - uj[1], ui[2] - uj[2]};
            const double eps = 0.01 * hij * hij;
            double fv = fp;
            if (a.alpha > 0.0) {                                                   // tv:432-448
                const double vr = vij[0] * xij[0] + vij[1] * xij[1] + vij[2] * xij[2];
                if (vr < 0.0) {
                    const double muij = hij * vr / (r2 + eps);
                    fv += mj * (a.alpha * a.c0 * muij) / (0.5 * (rhoi + rhoj));
                }
            }
#pragma unroll
            for (int d = 0; d < 3; d++) {
                v[d] += fv * dw[d];
                vh[d] += fh * dwh[d];
            }
            if (a.nu > 0.0) {                                                      // gtvf.py:274-288
                const double etai = a.nu * rhoi, etaj = a.nu * rhoj;
                const double etaij = 4.0 * (etai * etaj) / (etai + etaj);
                const double xd = dw[0] * xij[0] + dw[1] * xij[1] + dw[2] * xij[2];
                const double f = mj / (rhoi * rhoj) * etaij * xd / (r2 + eps);
#pragma unroll
                for (int d = 0; d < 3; d++) v[d] += f * vij[d];
            }
            if (fluid) {                                                           // gtvf.py:309-348
                const double di[3] = {uhi[0] - ui[0], uhi[1] - ui[1], uhi[2] - ui[2]};
                const double dj[3] = {a.uh[gj] - uj[0], a.vh[gj] - uj[1], a.wh[gj] - uj[2]};
#pragma unroll
                for (int i = 0; i < 3; i++) {
                    double res = 0.0;
#pragma unroll
                    for (int j = 0; j < 3; j++) res += (ui[i] * di[j] / rhoi + uj[i] * dj[j] / rhoj) * dw[j];
                    v[i] += mj * res;
                }
            }
        }
    });
    pairs_flush(a, npairs);
    if (!active) return;
    const uint32_t g = gi;
    if constexpr (PASS == GTVF_WALLV) {                                            // tv:119-134
        double uf[3] = {v[0], v[1], v[2]};
        if (s0 > 1e-12)
            for (int d = 0; d < 3; d++) uf[d] /= s0;
        a.wij[g] = (float)s0;
        a.uf[g] = (float)uf[0]; a.vf[g] = (float)uf[1]; a.wf[g] = (float)uf[2];
        a.ug[g] = 2.0 * a.u[g] - uf[0];
        a.vg[g] = 2.0 * a.v[g] - uf[1];
        a.wg[g] = 2.0 * a.w[g] - uf[2];
    } else if constexpr (PASS == GTVF_CONT) {
        a.arho[g] = (float)s0;
    } else if constexpr (PASS == GTVF_RHO) {                                       // gtvf.py:147-148
        const double rho = s0 / (s1 < 1.0 ? s1 : 1.0);
        a.rho[g] = rho;
        a.rhodiv[g] = s1;
        a.pf[g] = a.pref * (rho / a.rho0c - 1.0);                                  // tv:215-216
    } else if constexpr (PASS == GTVF_WALLP) {                                     // tv:730-736
        const double p = v[0] > 1e-14 ? s1 / v[0] : s1;
        a.vol[g] = (float)s0;
        a.wij[g] = (float)v[0];
        a.p[g] = (float)p;
        a.rho[g] = a.rho0c * (p / a.pref + 1.0);
    } else {
        // MomentumEquationPressureGradient.initialize sets au = g, and
        // MomentumEquationArtificialViscosity.initialize, which runs after it, zeroes it again:
        // with alpha > 0 the body force does not reach au (as in the reference)
        const double g0 = a.alpha > 0.0 ? 0.0 : a.gx, g1 = a.alpha > 0.0 ? 0.0 : a.gy, g2 = a.alpha > 0.0 ? 0.0 : a.gz;
        a.au[g] = (float)(g0 + v[0]); a.av[g] = (float)(g1 + v[1]); a.aw[g] = (float)(g2 + v[2]);
        a.auh[g] = (float)vh[0]; a.avh[g] = (float)vh[1]; a.awh[g] = (float)vh[2];
        a.p0[g] = p0i;
    }
}

// GTVFStep (gtvf.py:70-98) on the real particles of array `arr` (-1: every array):
//   1: u += dt/2 au, uhat = u + dt/2 auhat    2: rho += dt arho, x += dt uhat    3: u += dt/2 au
// (sigma += dt asigma adds zero: the scheme writes no asigma, and the host refuses arrays that
// carry one)
struct StageGtvfArgs {
    double *x, *y, *z, *u, *v, *w, *uh, *vh, *wh, *rho;
    const float *au, *av, *aw, *auh, *avh, *awh, *arho;
    const uint8_t *ptype;
    long long pool_end;
    unsigned mask;
    int which;
    double dt;
    const double *tc;
};
__global__ void k_stage_gtvf(const StageGtvfArgs a)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    const uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST) || !((a.mask >> (t & 7)) & 1u)) return;
    const double dt = a.tc ? a.tc[0] : a.dt;
    if (a.which == 2) {
        a.rho[g] += dt * (double)a.arho[g];
        a.x[g] += dt * a.uh[g];
        a.y[g] += dt * a.vh[g];
        a.z[g] += dt * a.wh[g];
        return;
    }
    const double dtb2 = 0.5 * dt;
    const double u = a.u[g] + dtb2 * (double)a.au[g];
    const double v = a.v[g] + dtb2 * (double)a.av[g];
    const double w = a.w[g] + dtb2 * (double)a.aw[g];
    a.u[g] = u; a.v[g] = v; a.w[g] = w;
    if (a.which == 1) {
        a.uh[g] = u + dtb2 * (double)a.auh[g];
        a.vh[g] = v + dtb2 * (double)a.avh[g];
        a.wh[g] = w + dtb2 * (double)a.awh[g];
    }
}
