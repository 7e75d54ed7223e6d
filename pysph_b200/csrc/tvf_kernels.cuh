// tvf_kernels.cuh -- EDAC / transport-velocity passes.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// EDAC scheme, transport-velocity branch (wc/edac.py:776-880): two passes over the same
// persistent neighbour lists.  Sorted records: AB = {A, B} as for k_pair_list,
// C2 = (rho, p, V, type) [ctx->C], Dv = (uhat-u, vhat-v, what-w, pavg), PT = (p, type)
// --------------------------------------------------------------------------
struct TvfArgs {
    const float4 *AB;
    float4 *C2, *Dv;
    const float2 *PT;
    const uint32_t *perm;
    double *rho;
    float *V, *pavg, *au, *av, *aw, *auhat, *avhat, *awhat, *ap;
    long long n;
    float cellx, celly, cellz, k2, kfac;
    unsigned fluid_mask, eqbits;
    int bql;
    float pb, nu, edac_nu, c0, alpha, gx, gy, gz;  // gx.. already damped
    unsigned long long *pair_counter;
    // solid walls (EDACScheme(fluids, solids), wc/edac.py:815-822): sources of the fluids' V,
    // average pressure, pressure gradient, artificial viscosity, no-slip term and EDAC
    // equation; destinations of k_tvf_wall.  src_mask = fluid_mask | solid_mask.
    unsigned solid_mask, src_mask;
    int avg_only;                 // k_tvf_pass1: only the average pressure, real destinations
    float wgx, wgy, wgz;          // the UNDAMPED body force of SolidWallPressureBC (:141-161)
    // the external-flow branch (pb == 0, wc/edac.py:882-971): XSPHCorrection(eps) with the fluid
    // itself as its only source, ClampWallPressure behind the wall pressure
    float eps_xsph;
    int clamp_p;
    float *ax, *ay, *az;
    float *p32;                   // pool p of the wall arrays
    double *ug, *vg, *wg;         // wall arrays: the slots of uhat vhat what hold ug vg wg,
    // ... those of auhat avhat awhat hold uf vf wf and pavg holds wij
};

__global__ void k_pack_tvf(const double *__restrict__ u, const double *__restrict__ v, const double *__restrict__ w,
                           const double *__restrict__ m, const double *__restrict__ uh, const double *__restrict__ vh,
                           const double *__restrict__ wh, const double *__restrict__ pf, const float *__restrict__ pavg,
                           const uint8_t *__restrict__ ptype, const uint32_t *__restrict__ perm, long long n,
                           float4 *__restrict__ B, float4 *__restrict__ AB, float4 *__restrict__ C2,
                           float4 *__restrict__ Dv, float2 *__restrict__ PT, const double *__restrict__ rho,
                           const unsigned solid_mask)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = perm[s];
    const int t = (int)ptype[g];
    const double ug = u[g], vg = v[g], wg = w[g];
    float4 b;
    b.x = (float)ug; b.y = (float)vg; b.z = (float)wg; b.w = (float)m[g];
    B[s] = b;
    AB[2 * s + 1] = b;
    // differences of nearly equal numbers: formed in fp64, then rounded
    Dv[s] = make_float4((float)(uh[g] - ug), (float)(vh[g] - vg), (float)(wh[g] - wg), pavg[g]);
    const float p = (float)pf[g];
    PT[s] = make_float2(p, __int_as_float(t));
    C2[s] = make_float4(0.f, p, 1.f, __int_as_float(t));   // rho, V filled in by pass 1
    if ((solid_mask >> (t & 7)) & 1u) {
        // a wall particle: its density is a constant of the run, p / V / the dummy velocity
        // come from k_tvf_wall
        C2[s] = make_float4((float)rho[g], 0.f, 1.f, __int_as_float(t));
        Dv[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// group 1 (real=False): V_i = sum_j W_ij, rho_i = m_i V_i (transport_velocity.py:52-58) and the
// neighbour-average pressure (wc/edac.py:69-79), every fluid particle incl. ghosts
template <int K, int DIM>
__global__ void __launch_bounds__(LIST_NT, 4) k_tvf_pass1(const TvfArgs a, const uint32_t *__restrict__ cnt,
                                                         const uint32_t *__restrict__ lst, const int capg)
{
    const int tid = threadIdx.x;
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * LIST_NT + tid;
    bool active = s < a.n;
    float4 Ai = make_float4(0.f, 0.f, 0.f, 0.f), Bi = Ai;
    int count = 0;
    if (active) {
        const int ti = __float_as_int(a.PT[s].y);
        if (!((a.fluid_mask >> (ti & 7)) & 1u)) active = false;
        if (a.avg_only && (ti & PT_GHOST)) active = false;   // that Group is real=True (wc/edac.py:842)
    }
    if (active) {
        ld_256(a.AB + 2 * (size_t)s, Ai, Bi);
        count = (int)cnt[s];
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *my = list_slot(lst, capg, s);
    const float hi2 = a.k2 * Ai.w * Ai.w;
    float wsum = 0.f, psum = 0.f, nn = 0.f;
    unsigned npairs = 0;
    struct Rec { float4 A; float2 P; };
    list_walk<Rec>(my, count, cmax,
        [&](const uint32_t e, Rec &r) {
            const uint32_t j = LIST_J(e);
            r.A = a.AB[2u * j];
            r.P = a.PT[j];
        },
        [&](const bool live, const uint32_t e, const Rec &r) {
            const float4 Aj = r.A;
            const float2 Pj = r.P;
            float xij, yij, zij;
            const float r2 = list_dist(e, a.cellx, a.celly, a.cellz, Ai, Aj, xij, yij, zij);
            if (live && NNPS_ACCEPT(r2, hi2, a.k2, Aj.w) && ((a.src_mask >> (__float_as_int(Pj.y) & 7)) & 1u)) {
                npairs++;
                const float rij = sqrtf(r2);
                const float h1 = frcp(0.5f * (Ai.w + Aj.w));
                float w, dw;
                sph_kernel<K>(rij * h1, w, dw);
                wsum += w * a.kfac * hpow<DIM>(h1);
                psum += Pj.x;
                nn += 1.0f;
            }
        });
    if (active) {
        const uint32_t g = a.perm[s];
        if (!a.avg_only) {
            const float rho = Bi.w * wsum;
            a.V[g] = wsum;
            a.rho[g] = (double)rho;
            float4 *c2 = a.C2 + s;
            c2->x = rho;          // .y (p) and .w (type) were written by k_pack_tvf; other
            c2->z = wsum;         // threads read only those two while this kernel runs
        }
        if (a.bql) {
            const float pv = nn > 0.f ? psum / nn : 0.f;
            a.pavg[g] = pv;
            a.Dv[s].w = pv;
        }
    }
    pairs_flush(a, npairs);
}

// group 1, the wall arrays (real=False; wc/edac.py:815-822), after k_tvf_pass1 has put the
// fluids' new density into their records: SourceNumberDensity (:177-183: wij = sum over the
// FLUID neighbours of W), VolumeSummation (transport_velocity.py:61-75: V = sum over ALL
// neighbours), SolidWallPressureBC (:136-166: p = sum_f (p_f + rho_f (g - a_wall) . x_wf) W / wij)
// and SetWallVelocity (:186-230: uf = sum_f u_f W / wij, ug = 2 u_wall - uf).  Results go to the
// pool (p; V; wij, uf.., ug.. in the transport-velocity slots a wall does not use) and into the
// wall particle's own records, from which group 2 reads them as a SOURCE: C2 = (rho, p, V, type),
// Dv = (ug, vg, wg, -), PT = (p, type).
template <int K, int DIM>
__global__ void __launch_bounds__(LIST_NT, 4) k_tvf_wall(const TvfArgs a, const uint32_t *__restrict__ cnt,
                                                        const uint32_t *__restrict__ lst, const int capg)
{
    const int tid = threadIdx.x;
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * LIST_NT + tid;
    bool active = s < a.n;
    float4 Ai = make_float4(0.f, 0.f, 0.f, 0.f), Bi = Ai;
    int count = 0;
    int ti = 0;
    if (active) {
        ti = __float_as_int(a.PT[s].y);
        if (!((a.solid_mask >> (ti & 7)) & 1u)) active = false;
    }
    uint32_t g = 0;
    float gax = 0.f, gay = 0.f, gaz = 0.f;
    if (active) {
        ld_256(a.AB + 2 * (size_t)s, Ai, Bi);
        count = (int)cnt[s];
        g = a.perm[s];
        // g - a_wall: au av aw of a wall array are its PRESCRIBED acceleration
        gax = a.wgx - a.au[g]; gay = a.wgy - a.av[g]; gaz = a.wgz - a.aw[g];
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *my = list_slot(lst, capg, s);
    const float hi2 = a.k2 * Ai.w * Ai.w;
    float vsum = 0.f, wsum = 0.f, psum = 0.f, us = 0.f, vs = 0.f, ws = 0.f;
    unsigned npairs = 0;
    struct Rec { float4 A, B, C; };
    list_walk<Rec>(my, count, cmax,
        [&](const uint32_t e, Rec &r) {
            const uint32_t j = LIST_J(e);
            ld_256(a.AB + 2u * j, r.A, r.B);
            r.C = a.C2[j];      // a fluid's (rho, p, ., type); of a wall only the type is used
        },
        [&](const bool live, const uint32_t e, const Rec &r) {
            const float4 Aj = r.A, Bj = r.B, Cj = r.C;
            float xij, yij, zij;
            const float r2 = list_dist(e, a.cellx, a.celly, a.cellz, Ai, Aj, xij, yij, zij);
            const int tj = __float_as_int(Cj.w) & 7;
            if (live && NNPS_ACCEPT(r2, hi2, a.k2, Aj.w) && ((a.src_mask >> tj) & 1u)) {
                npairs++;
                const float rij = sqrtf(r2);
                const float h1 = frcp(0.5f * (Ai.w + Aj.w));
                float w, dw;
                sph_kernel<K>(rij * h1, w, dw);
                w *= a.kfac * hpow<DIM>(h1);
                vsum += w;
                if ((a.fluid_mask >> tj) & 1u) {
                    wsum += w;
                    psum += (Cj.y + Cj.x * (gax * xij + gay * yij + gaz * zij)) * w;
                    us += Bj.x * w; vs += Bj.y * w; ws += Bj.z * w;
                }
            }
        });
    if (active) {
        float pw = wsum > 1e-14f ? psum / wsum : psum;
        if (a.clamp_p && pw < 0.f) pw = 0.f;               // ClampWallPressure wc/edac.py:169-174
        if (wsum > 1e-12f) {
            const float w1 = 1.0f / wsum;
            us *= w1; vs *= w1; ws *= w1;
        }
        const float ug = 2.0f * Bi.x - us, vg = 2.0f * Bi.y - vs, wg = 2.0f * Bi.z - ws;
        a.V[g] = vsum;
        a.p32[g] = pw;
        a.pavg[g] = wsum;                                      // wij
        a.auhat[g] = us; a.avhat[g] = vs; a.awhat[g] = ws;     // uf vf wf
        a.ug[g] = (double)ug; a.vg[g] = (double)vg; a.wg[g] = (double)wg;
        float4 *c2 = a.C2 + s;
        c2->y = pw;           // .x (rho) and .w (type) stay; other threads read a wall's .w only
        c2->z = vsum;
        a.Dv[s] = make_float4(ug, vg, wg, 0.f);
        float2 *pt = const_cast<float2 *>(a.PT) + s;
        pt->x = pw;
    }
    pairs_flush(a, npairs);
}

// group 2 (real=True): pressure gradient with the background-pressure term, artificial /
// physical viscosity, artificial stress and the EDAC pressure evolution, fused.  WALLS: solid
// walls are sources too -- of the pressure gradient, the artificial viscosity, the EDAC
// equation and (instead of the viscosity) SolidWallNoSlipBC, which takes the dummy velocity
// from the wall's Dv record; the instantiation without walls is the measured one.
// EXT (implies WALLS): the external-flow branch -- the number-density MomentumEquation
// (wc/edac.py:301-352: the pressure gradient without average and background pressure) and
// XSPHCorrection (basic_equations.py:260-300) over the destination's own array.
template <int K, int DIM, bool WALLS = false, bool EXT = false>
__global__ void __launch_bounds__(LIST_NT, 6) k_tvf_pass2(const TvfArgs a, const uint32_t *__restrict__ cnt,
                                                         const uint32_t *__restrict__ lst, const int capg)
{
    const int tid = threadIdx.x;
    const unsigned FULL = 0xffffffffu;
    const long long s = (long long)blockIdx.x * LIST_NT + tid;
    bool active = s < a.n;
    float4 Ai = make_float4(0.f, 0.f, 0.f, 0.f), Bi = Ai, Ci = make_float4(1.f, 0.f, 1.f, 0.f), Di = Ai;
    int count = 0;
    if (active) {
        Ci = a.C2[s];
        const int ti = __float_as_int(Ci.w);
        if ((ti & PT_GHOST) || !((a.fluid_mask >> (ti & 7)) & 1u)) active = false;
    }
    if (active) {
        ld_256(a.AB + 2 * (size_t)s, Ai, Bi);
        Di = a.Dv[s];
        count = (int)cnt[s];
    }
    int cmax = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(FULL, cmax, o));
    const uint32_t *my = list_slot(lst, capg, s);
    const float hi2 = a.k2 * Ai.w * Ai.w;
    const float rhoi = Ci.x, pi = Ci.y, pavg = Di.w;
    const float Vi1 = frcp(Ci.z);
    const float Vi2 = Vi1 * Vi1;
    const float mi1 = frcp(Bi.w);
    const float cs2 = a.c0 * a.c0;
    float au = 0.f, av = 0.f, aw = 0.f, auh = 0.f, avh = 0.f, awh = 0.f, ap = 0.f;
    float xs = 0.f, ys = 0.f, zs = 0.f;          // XSPH sums (EXT)
    const int ti7 = __float_as_int(Ci.w) & 7;
    unsigned npairs = 0;
    struct Rec { float4 A, B, C, D; };
    list_walk<Rec>(my, count, cmax,
        [&](const uint32_t e, Rec &r) {
            const uint32_t j = LIST_J(e);
            ld_256(a.AB + 2u * j, r.A, r.B);
            r.C = a.C2[j];
            r.D = a.Dv[j];
        },
        [&](const bool live, const uint32_t e, const Rec &r) {
            const float4 Aj = r.A, Bj = r.B, Cj = r.C, Dj = r.D;
            float xij, yij, zij;
            const float r2 = list_dist(e, a.cellx, a.celly, a.cellz, Ai, Aj, xij, yij, zij);
            const int tj = __float_as_int(Cj.w) & 7;
            const bool wall = WALLS && ((a.solid_mask >> tj) & 1u);
            if (live && NNPS_ACCEPT(r2, hi2, a.k2, Aj.w) && (((WALLS ? a.src_mask : a.fluid_mask) >> tj) & 1u)) {
                npairs++;
                const bool far = r2 > 1e-24f;
                const float rinv = far ? frsqrt(r2) : 0.0f;
                const float rij = r2 * rinv;
                const float hij = 0.5f * (Ai.w + Aj.w);
                const float h1 = frcp(hij);
                float w, dw;
                sph_kernel<K>(rij * h1, w, dw);
                const float gt = dw * a.kfac * hpow<DIM>(h1) * h1 * rinv;   // DWIJ = gt * XIJ
                const float eps = 0.01f * hij * hij;
                const float rhoj = Cj.x, pj = Cj.y;
                const float Vj1 = frcp(Cj.z);
                const float common = mi1 * (Vi2 + Vj1 * Vj1);
                const float uij = Bi.x - Bj.x, vij = Bi.y - Bj.y, wij = Bi.z - Bj.z;
                const float vdotx = uij * xij + vij * yij + wij * zij;
                const float rsum1 = frcp(rhoi + rhoj);
                const float r2e1 = frcp(r2 + eps);
                float fx = 0.f;   // multiplies XIJ in au
                if (EXT && (a.eqbits & B200SPH_TVF_MOM)) {   // wc/edac.py:319-341
                    const float pij = (rhoj * pi + rhoi * pj) * rsum1;
                    fx += -pij * common * gt;
                }
                if (EXT && (a.eqbits & B200SPH_TVF_XSPH) && tj == ti7) {   // basic_equations.py:285-295
                    const float t_ = -a.eps_xsph * Bj.w * (w * a.kfac * hpow<DIM>(h1)) * (2.0f * rsum1);
                    xs += t_ * uij; ys += t_ * vij; zs += t_ * wij;
                }
                if (a.eqbits & B200SPH_TVF_PGRAD) {   // wc/edac.py:447-481
                    const float pij = (rhoj * (pi - pavg) + rhoi * (pj - pavg)) * rsum1;
                    fx += -pij * common * gt;
                    const float fh = -a.pb * common * gt;
                    auh += fh * xij;
                    avh += fh * yij;
                    awh += fh * zij;
                }
                if ((a.eqbits & B200SPH_TVF_AV) && vdotx < 0.f) {   // transport_velocity.py:432-448
                    const float muij = hij * vdotx * r2e1;
                    const float piij = Bj.w * (-a.alpha * a.c0 * muij) * (2.0f * rsum1);
                    fx += -piij * gt;
                }
                au += fx * xij;
                av += fx * yij;
                aw += fx * zij;
                if ((a.eqbits & B200SPH_TVF_VISC) && !wall) {   // transport_velocity.py:362-386
                    const float etaij = 2.0f * a.nu * rhoi * rhoj * rsum1;
                    const float tmp = common * etaij * (gt * r2) * r2e1;
                    au += tmp * uij;
                    av += tmp * vij;
                    aw += tmp * wij;
                }
                if (WALLS && wall && (a.eqbits & B200SPH_TVF_NOSLIP)) {   // transport_velocity.py:611-638
                    const float etaij = 2.0f * a.nu * rhoi * rhoj * rsum1;
                    const float tmp = common * etaij * (gt * r2) * r2e1;
                    au += tmp * (Bi.x - Dj.x);      // the wall's dummy velocity ug vg wg
                    av += tmp * (Bi.y - Dj.y);
                    aw += tmp * (Bi.z - Dj.z);
                }
                if ((a.eqbits & B200SPH_TVF_ASTRESS) && !wall) {   // transport_velocity.py:473-545
                    const float si = rhoi * gt * (Di.x * xij + Di.y * yij + Di.z * zij);
                    const float sj = rhoj * gt * (Dj.x * xij + Dj.y * yij + Dj.z * zij);
                    const float c = 0.5f * common;
                    au += c * (Bi.x * si + Bj.x * sj);
                    av += c * (Bi.y * si + Bj.y * sj);
                    aw += c * (Bi.z * si + Bj.z * sj);
                }
                if (a.eqbits & B200SPH_TVF_EDAC) {   // wc/edac.py:365-386
                    const float etaij = 2.0f * a.edac_nu * rhoi * rhoj * rsum1;
                    ap += rhoi * frcp(rhoj) * cs2 * Bj.w * (gt * vdotx);
                    ap += common * etaij * (gt * r2) * r2e1 * (pi - pj);
                }
            }
        });
    if (active) {
        const uint32_t g = a.perm[s];
        if (a.eqbits & B200SPH_TVF_PGRAD) {   // post_loop wc/edac.py:483-488
            au += a.gx; av += a.gy; aw += a.gz;
            a.auhat[g] = auh; a.avhat[g] = avh; a.awhat[g] = awh;
        }
        if (EXT && (a.eqbits & B200SPH_TVF_MOM)) {   // post_loop wc/edac.py:343-352
            au += a.gx; av += a.gy; aw += a.gz;
        }
        if (EXT && (a.eqbits & B200SPH_TVF_XSPH)) {  // post_loop basic_equations.py:297-300
            a.ax[g] = xs + Bi.x; a.ay[g] = ys + Bi.y; a.az[g] = zs + Bi.z;
        }
        a.au[g] = au; a.av[g] = av; a.aw[g] = aw;
        if (a.eqbits & B200SPH_TVF_EDAC) a.ap[g] = ap;
    }
    pairs_flush(a, npairs);
}

struct StageTvfArgs {
    double *x, *y, *z, *u, *v, *w, *pf, *uh, *vh, *wh;
    double *x0, *y0, *z0, *u0, *v0, *w0, *pf0;
    const float *au, *av, *aw, *auh, *avh, *awh, *ap;
    const uint8_t *ptype;
    long long pool_end;
    int arr, which;
    double f;
    const double *tc;                // device-resident dt (tc[0]); null: f
    // EDACStep (wc/edac.py:82-133, the scheme without transport velocity): positions move with
    // the XSPH-corrected velocity ax ay az, there is no uhat
    int ext;
    const float *ax, *ay, *az;
};
// EDACTVFStep wc/edac.py:491-540 / EDACStep :82-133 (real particles)
__device__ __forceinline__ void stage_tvf_body(const StageTvfArgs &a)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST)) return;
    if (a.arr >= 0 && (t & 7) != a.arr) return;
    if (a.which == 0) {
        a.x0[g] = a.x[g]; a.y0[g] = a.y[g]; a.z0[g] = a.z[g];
        a.u0[g] = a.u[g]; a.v0[g] = a.v[g]; a.w0[g] = a.w[g];
        a.pf0[g] = a.pf[g];
        return;
    }
    const double f = stage_factor(a.tc, a.f, a.which, false);
    const double u = a.u0[g] + f * (double)a.au[g];
    const double v = a.v0[g] + f * (double)a.av[g];
    const double w = a.w0[g] + f * (double)a.aw[g];
    a.u[g] = u; a.v[g] = v; a.w[g] = w;
    if (a.ext) {
        a.x[g] = a.x0[g] + f * (double)a.ax[g];
        a.y[g] = a.y0[g] + f * (double)a.ay[g];
        a.z[g] = a.z0[g] + f * (double)a.az[g];
    } else {
        const double uh = u + f * (double)a.auh[g];
        const double vh = v + f * (double)a.avh[g];
        const double wh = w + f * (double)a.awh[g];
        a.uh[g] = uh; a.vh[g] = vh; a.wh[g] = wh;
        a.x[g] = a.x0[g] + f * uh;
        a.y[g] = a.y0[g] + f * vh;
        a.z[g] = a.z0[g] + f * wh;
    }
    a.pf[g] = a.pf0[g] + f * (double)a.ap[g];
}
__global__ void k_stage_tvf(StageTvfArgs a) { stage_tvf_body(a); }
