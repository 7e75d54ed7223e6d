// pool_kernels.cuh -- elementwise / reduction kernels over the particle pool.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// elementwise / reduction kernels over the pool
// --------------------------------------------------------------------------
struct PoolLayout {
    int narr;
    long long off[B200SPH_MAX_ARRAYS], n[B200SPH_MAX_ARRAYS], n_real[B200SPH_MAX_ARRAYS];
};

__global__ void k_fill_ptype(uint8_t *ptype, long long pool_end, PoolLayout L)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= pool_end) return;
    uint8_t t = PT_INVALID;
    for (int a = 0; a < L.narr; a++) {
        long long i = g - L.off[a];
        if (i >= 0 && i < L.n[a]) t = (uint8_t)(a | (i >= L.n_real[a] ? PT_GHOST : 0));
    }
    ptype[g] = t;
}

__global__ void k_red_init(long long *red)
{
    int i = threadIdx.x;
    if (i < 16) red[i] = (i & 1) ? d2o(-1e300) : d2o(1e300);  // even: min slots, odd: max slots
}

// slots: 0 xmin 1 xmax 2 ymin 3 ymax 4 zmin 5 zmax 6 hmin 7 hmax
__global__ void k_reduce_minmax(const double *__restrict__ x, const double *__restrict__ y,
                                const double *__restrict__ z, const double *__restrict__ h,
                                const uint8_t *__restrict__ ptype, long long pool_end,
                                int do_xyz, int do_h, long long *red)
{
    double mn[4] = {1e300, 1e300, 1e300, 1e300}, mx[4] = {-1e300, -1e300, -1e300, -1e300};
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < pool_end;
         g += (long long)gridDim.x * blockDim.x) {
        if (ptype[g] == PT_INVALID) continue;
        if (do_xyz) {
            double v = x[g]; mn[0] = fmin(mn[0], v); mx[0] = fmax(mx[0], v);
            v = y[g]; mn[1] = fmin(mn[1], v); mx[1] = fmax(mx[1], v);
            v = z[g]; mn[2] = fmin(mn[2], v); mx[2] = fmax(mx[2], v);
        }
        if (do_h) {
            double v = h[g]; mn[3] = fmin(mn[3], v); mx[3] = fmax(mx[3], v);
        }
    }
    for (int k = 0; k < 4; k++) {
        for (int o = 16; o > 0; o >>= 1) {
            mn[k] = fmin(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
            mx[k] = fmax(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 4; k++) {
            if ((k < 3 && !do_xyz) || (k == 3 && !do_h)) continue;
            atomicMin(&red[2 * k], d2o(mn[k]));
            atomicMax(&red[2 * k + 1], d2o(mx[k]));
        }
    }
}

// slots: 9 max dt_cfl, 11 max dt_force (real particles), 12 min h (all)
__global__ void k_reduce_dt(const float *__restrict__ dt_cfl, const float *__restrict__ dt_force,
                            const double *__restrict__ h, const uint8_t *__restrict__ ptype,
                            long long pool_end, long long *red)
{
    double mc = -1e300, mf = -1e300, hm = 1e300;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < pool_end;
         g += (long long)gridDim.x * blockDim.x) {
        uint8_t t = ptype[g];
        if (t == PT_INVALID) continue;
        hm = fmin(hm, h[g]);
        if (t & PT_GHOST) continue;
        mc = fmax(mc, (double)dt_cfl[g]);
        mf = fmax(mf, (double)dt_force[g]);
    }
    for (int o = 16; o > 0; o >>= 1) {
        mc = fmax(mc, __shfl_xor_sync(0xffffffffu, mc, o));
        mf = fmax(mf, __shfl_xor_sync(0xffffffffu, mf, o));
        hm = fmin(hm, __shfl_xor_sync(0xffffffffu, hm, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&red[9], d2o(mc));
        atomicMax(&red[11], d2o(mf));
        atomicMin(&red[12], d2o(hm));
    }
}

// Integrator.compute_time_step (integrator.py:161-200) on the reduced factors: the local
// proposal cfl * dt_min, or 1e20 when no factor constrains it (solver.py:655-660)
__device__ __forceinline__ void dt_propose(const long long *red, double *tc, const double cfl, const int fixed_h)
{
    const double mc = o2d(red[9]), mf = o2d(red[11]);
    const double f_cfl = mc < -1e299 ? -1.0 : mc, f_force = mf < -1e299 ? -1.0 : mf;
    double hmin = fmin(1.0, o2d(red[12]));
    if (!fixed_h || tc[3] < 0.0) tc[3] = hmin;
    hmin = tc[3];
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    double dt_cfl = inf, dt_force = inf;
    if (f_cfl > 0.0) dt_cfl = hmin / f_cfl;
    if (f_force > 0.0) dt_force = sqrt(hmin / sqrt(f_force));
    const double dt_min = fmin(dt_cfl, dt_force);
    tc[2] = (dt_min <= 0.0 || isinf(dt_min)) ? 1e20 : cfl * dt_min;
}
// Solver loop bookkeeping (solver.py:478-491, :647-688): t += dt; dt = damp(new dt)
// and the last step lands on the final time (solver.py:757-760, :771-773)
__device__ __forceinline__ void dt_commit(double *tc, const double prev_factor, const double new_factor, const int in_parallel,
                                          const int adaptive, const int advance, const double t_final, const double t_eps)
{
    const double dt_old = tc[0];
    if (advance) tc[1] += dt_old;
    const double t = tc[1];
    if (fabs(t_final - t) < t_eps) return;  // reached the end: dt stays
    const double undamped = dt_old / prev_factor;
    double dt = undamped;
    if (adaptive) {
        dt = tc[2];
        if (!in_parallel && dt >= 1e20) dt = undamped;
    }
    dt *= new_factor;
    if (t + dt > t_final - t_eps) dt = t_final - t;
    tc[0] = dt;
}
// the slots are re-armed for the next reduction (the fused stage kernel adds to them directly)
__global__ void k_dt_propose(long long *__restrict__ red, double *__restrict__ tc, double cfl, int fixed_h)
{
    dt_propose(red, tc, cfl, fixed_h);
    red[9] = d2o(-1e300); red[11] = d2o(-1e300); red[12] = d2o(1e300);
}
__global__ void k_dt_commit(double *__restrict__ tc, double prev_factor, double new_factor, int in_parallel, int adaptive, int advance,
                            double t_final, double t_eps)
{
    dt_commit(tc, prev_factor, new_factor, in_parallel, adaptive, advance, t_final, t_eps);
}
// both in one launch (one rank: nothing to reduce in between)
__global__ void k_dt_advance(long long *__restrict__ red, double *__restrict__ tc, double cfl, int fixed_h,
                             double prev_factor, double new_factor, int adaptive, int advance, double t_final, double t_eps)
{
    if (adaptive) dt_propose(red, tc, cfl, fixed_h);
    red[9] = d2o(-1e300); red[11] = d2o(-1e300); red[12] = d2o(1e300);
    dt_commit(tc, prev_factor, new_factor, 0, adaptive, advance, t_final, t_eps);
}
// UpdateSmoothingLengthFerrari.loop wc/basic.py:458-463
__global__ void k_ferrari(double *__restrict__ h, const double *__restrict__ m,
                          const double *__restrict__ rho, long long lo, long long hi, double hdx,
                          double dim1)
{
    long long g = lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= hi) return;
    h[g] = hdx * pow(m[g] / rho[g], dim1);
}

struct StageArgs {
    double *x, *y, *z, *u, *v, *w, *rho;
    double *x0, *y0, *z0, *u0, *v0, *w0, *rho0;
    const float *au, *av, *aw, *ax, *ay, *az, *arho;
    const uint8_t *ptype;
    long long pool_end;
    int arr, which;
    double f;
    const double *tc;                // device-resident dt (tc[0]); null: f
};

// WCSPHStep.stage1 / stage2 (integrator_step.py:63-91) for one property.  k_stage and
// k_stage_pack both go through wcsph_combine, so that both contract it to the same FMA.
__device__ __forceinline__ double wcsph_combine(const double q0, const double f, const float aq)
{
    return q0 + f * (double)aq;
}
// WCSPHTVDRK3Step.stage1 / stage2 / stage3 (integrator_step.py:118-168) for one property, in the
// reference's association order (rk3_combine, on the current value qc); rk3_update reads q[g]
// for stages 2 and 3 only.  k_stage_rk3 and k_stage_pack_rk3 both go through rk3_combine, so that
// both contract it to the same FMAs (k_stage_pack_rk3 passes rho after the pool-side EOS clamp).
__device__ __forceinline__ double rk3_combine(const int which, const double q0, const double qc, const double dt,
                                              const float aq)
{
    if (which == 1) return q0 + dt * (double)aq;
    if (which == 2) return 0.75 * q0 + 0.25 * (qc + dt * (double)aq);
    return (1. / 3.) * q0 + (2. / 3.) * (qc + dt * (double)aq);
}
__device__ __forceinline__ double rk3_update(const int which, const double q0, const double *q,
                                             const long long g, const double dt, const float aq)
{
    return rk3_combine(which, q0, which == 1 ? 0.0 : q[g], dt, aq);
}

// WCSPHStep.initialize / stage1 / stage2 integrator_step.py:51-91 (real particles only,
// integrator_cython.mako:97-111)
__device__ __forceinline__ void stage_body(const StageArgs &a)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST)) return;
    if (a.arr >= 0 && (t & 7) != a.arr) return;
    if (a.which == 0) {
        a.x0[g] = a.x[g]; a.y0[g] = a.y[g]; a.z0[g] = a.z[g];
        a.u0[g] = a.u[g]; a.v0[g] = a.v[g]; a.w0[g] = a.w[g];
        a.rho0[g] = a.rho[g];
    } else {
        const double f = stage_factor(a.tc, a.f, a.which, false);
        a.u[g] = wcsph_combine(a.u0[g], f, a.au[g]);
        a.v[g] = wcsph_combine(a.v0[g], f, a.av[g]);
        a.w[g] = wcsph_combine(a.w0[g], f, a.aw[g]);
        a.x[g] = wcsph_combine(a.x0[g], f, a.ax[g]);
        a.y[g] = wcsph_combine(a.y0[g], f, a.ay[g]);
        a.z[g] = wcsph_combine(a.z0[g], f, a.az[g]);
        a.rho[g] = wcsph_combine(a.rho0[g], f, a.arho[g]);
    }
}
__global__ void k_stage(StageArgs a) { stage_body(a); }

// WCSPHTVDRK3Step stage1 / stage2 / stage3 (a.which = 1, 2, 3), real particles only;
// its initialize is WCSPHStep's (k_stage, which = 0)
__device__ __forceinline__ void stage_rk3_body(const StageArgs &a)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST)) return;
    if (a.arr >= 0 && (t & 7) != a.arr) return;
    const double dt = stage_factor(a.tc, a.f, a.which, true);
    a.u[g] = rk3_update(a.which, a.u0[g], a.u, g, dt, a.au[g]);
    a.v[g] = rk3_update(a.which, a.v0[g], a.v, g, dt, a.av[g]);
    a.w[g] = rk3_update(a.which, a.w0[g], a.w, g, dt, a.aw[g]);
    a.x[g] = rk3_update(a.which, a.x0[g], a.x, g, dt, a.ax[g]);
    a.y[g] = rk3_update(a.which, a.y0[g], a.y, g, dt, a.ay[g]);
    a.z[g] = rk3_update(a.which, a.z0[g], a.z, g, dt, a.az[g]);
    a.rho[g] = rk3_update(a.which, a.rho0[g], a.rho, g, dt, a.arho[g]);
}
__global__ void k_stage_rk3(StageArgs a) { stage_rk3_body(a); }

// the pending equation-of-state calls on the pool (eos_tab_eval, the clamped rho written back)
__device__ __forceinline__ void eos_tab_apply(double *__restrict__ rho, float *__restrict__ p, float *__restrict__ cs,
                                              const uint8_t t, const long long g, const EosTab &E)
{
    if (!eos_tab_applies(E, t)) return;
    double r = rho[g];
    float pg, csg;
    if (eos_tab_eval(E, t & 7, r, pg, csg)) rho[g] = r;
    p[g] = pg;
    cs[g] = csg;
}

// ---------------------------------------------------------------------------
// The fused stage kernels of the WCSPH fast path (every array steps with WCSPHStep:
// k_stage_pack, or with WCSPHTVDRK3Step: k_stage_pack_rk3; the neighbour lists of the current
// build are reusable): in ONE pass over the pool, per real particle,
//   [initialize (integrator_step.py:51-61) when it was deferred to here: the copies take the
//    rho of before the EOS calls below, as the reference's initialize, which runs before them;
//    with INIT_RENAMED there is nothing to copy, x0 .. rho0 are that state already]
//   [the pool side of the last evaluation's EOS calls (k_eos_tab's arithmetic) when the pair
//    pass left it to here: rho clamp, p, cs -- ghosts included, as k_eos_tab]
//   stage1 / stage2 (integrator_step.py:63-91), fp64, wcsph_combine as k_stage
//     (k_stage_pack_rk3: stage1 / stage2 / stage3, :118-168, rk3_combine as k_stage_rk3)
//   the packed pair records of the NEXT evaluation at the particle's sorted slot:
//     {A, B} = (cell-relative position of the frozen build, h, u, v, w, m)   -- pack_position
//     C      = (rho, p / rho^2, cs, type) with the equation-of-state calls of the LAST
//              evaluation applied to the record only (eos_tab_eval, state_record); the pool's
//              rho / p / cs are written when the evaluation really issues those calls
//   the drift of the build (max |x - x_build|^2, max (h - h_build)) into red_u32
//   [the stepper's last stage: the adaptive-dt factors max dt_cfl, max dt_force, min h into
//    red[9,11,12]]
// It replaces k_stage(initialize) + k_eos_tab + k_stage + k_pack_pos_light + k_pack_state
// (+ k_reduce_dt): six sweeps over the fp64 state become one.  Ghost particles are not stepped
// (integrator_cython.mako:97-111) and their records are refreshed by the halo scatter.
// ---------------------------------------------------------------------------
// how the launch takes a deferred initialize (init_materialise): there is none; it copies
// x .. rho into x0 .. rho0 as it goes; or the host renamed the buffers (init_by_rename), so
// that a.x0 .. a.rho0 are the state before the stage and a.x .. a.rho only receive the new one
enum { INIT_NONE = 0, INIT_COPY = 1, INIT_RENAMED = 2 };

struct FusePackArgs {
    const double *h, *m;             // h null: every particle has h_uniform (the 32-byte records need that)
    double h_uniform;
    float *p, *cs;                   // pool values: read for arrays without a speculated EOS, written by EP
    const uint32_t *rank, *key_of;   // pool index -> sorted slot / cell key of the current build
    const float4 *A0;                // packed positions at build time (sorted order)
    float4 *AB, *C;
    float4 *R;                       // non-null: the state goes into the 32-byte records ...
    Rec32Eos E32;                    // ... formed with this EOS
    GridDev G;
    unsigned *red_u32;
    const float *dt_cfl, *dt_force;
    long long *red;
    int do_init, reduce_dt, eos_any; // do_init: INIT_*
    EosTab E;
    int eos_pool;                    // apply EP to the pool's rho / p / cs first
    EosTab EP;
    int half_pending;                // WCSPHStep stage 1: x .. rho and EP's p / cs are left to half_materialise
    // WCSPHStep stage 2 after such a stage 1: the predicted rho its EOS calls read is formed again
    // from rho0, stage 1's factor f_half and the first evaluation's arho (arho_half), as stage 1 did
    const float *arho_half;
    double f_half;
};

// The body of the fused stage kernels, the stage being WCSPHStep's or, RK3, WCSPHTVDRK3Step's.
// s_* is the kernel's shared memory of the block reduction (one atomic per block and quantity).
template <bool RK3>
__device__ __forceinline__ void stage_pack_body(const StageArgs &a, const FusePackArgs &q, float *s_d2, float *s_dh,
                                                double *s_mc, double *s_mf, double *s_hm)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float d2 = 0.f, dh = 0.f;
    double mc = -1e300, mf = -1e300, hm = 1e300;
    const uint8_t t = g < a.pool_end ? a.ptype[g] : (uint8_t)PT_INVALID;
    // (with the type, not behind it: one round trip to memory less before A0[s] can be asked for;
    // both arrays have a slot for every slot of the pool)
    const uint32_t s = g < a.pool_end ? q.rank[g] : 0u, key = g < a.pool_end ? q.key_of[g] : 0u;
    if (t != PT_INVALID) {
        const double hg = q.h ? q.h[g] : q.h_uniform;
        hm = hg;
        if (t & PT_GHOST) {
            if (q.eos_pool) eos_tab_apply(a.rho, q.p, q.cs, t, g, q.EP);
        } else {
            const double f = stage_factor(a.tc, a.f, a.which, RK3);
            // rho before the stage: the deferred initialize copies it as it is, the pool side of
            // the EOS calls clamps it; the stage overwrites the pool's rho, so only TVD-RK3's
            // stages 2 and 3 read the clamped value
            const bool eos = q.eos_pool && eos_tab_applies(q.EP, t);
            double x0, y0, z0, u0, v0, w0, r0;
            if (q.do_init == INIT_COPY) {
                x0 = a.x[g]; y0 = a.y[g]; z0 = a.z[g];
                u0 = a.u[g]; v0 = a.v[g]; w0 = a.w[g];
                r0 = a.rho[g];
                a.x0[g] = x0; a.y0[g] = y0; a.z0[g] = z0;
                a.u0[g] = u0; a.v0[g] = v0; a.w0[g] = w0;
                a.rho0[g] = r0;
            } else {   // (INIT_RENAMED: the state the initialize saw already goes by x0 .. rho0)
                x0 = a.x0[g]; y0 = a.y0[g]; z0 = a.z0[g];
                u0 = a.u0[g]; v0 = a.v0[g]; w0 = a.w0[g];
                r0 = a.rho0[g];
            }
            double rc = r0;
            if (!RK3 && q.arho_half) {
                if (eos) rc = wcsph_combine(r0, stage_factor(a.tc, q.f_half, 1, false), q.arho_half[g]);
            } else if (q.do_init == INIT_NONE && (eos || (RK3 && a.which != 1))) {
                rc = a.rho[g];
            }
            float p_eos = 0.f, cs_eos = 0.f;
            const bool store = RK3 || !q.half_pending;
            if (eos) {
                eos_tab_eval(q.EP, t & 7, rc, p_eos, cs_eos);
                if (store) {
                    q.p[g] = p_eos;
                    q.cs[g] = cs_eos;
                }
            }
            double un, vn, wn, xn, yn, zn, r;
            if (RK3) {
                un = rk3_update(a.which, u0, a.u, g, f, a.au[g]);
                vn = rk3_update(a.which, v0, a.v, g, f, a.av[g]);
                wn = rk3_update(a.which, w0, a.w, g, f, a.aw[g]);
                xn = rk3_update(a.which, x0, a.x, g, f, a.ax[g]);
                yn = rk3_update(a.which, y0, a.y, g, f, a.ay[g]);
                zn = rk3_update(a.which, z0, a.z, g, f, a.az[g]);
                r = rk3_combine(a.which, r0, rc, f, a.arho[g]);
            } else {
                un = wcsph_combine(u0, f, a.au[g]);
                vn = wcsph_combine(v0, f, a.av[g]);
                wn = wcsph_combine(w0, f, a.aw[g]);
                xn = wcsph_combine(x0, f, a.ax[g]);
                yn = wcsph_combine(y0, f, a.ay[g]);
                zn = wcsph_combine(z0, f, a.az[g]);
                r = wcsph_combine(r0, f, a.arho[g]);
            }
            if (store) {
                a.u[g] = un; a.v[g] = vn; a.w[g] = wn;
                a.x[g] = xn; a.y[g] = yn; a.z[g] = zn;
                a.rho[g] = r;
            }
            if (q.reduce_dt) {
                mc = (double)q.dt_cfl[g];
                mf = (double)q.dt_force[g];
            }
            // ---- records of the next evaluation ---------------------------------------
            const float4 A = pack_position(q.G, key, xn, yn, zn, hg);
            const int ar = t & 7;
            if (q.R) {
                // only the full sector: a lone 16-byte half would cost a read-modify-write in
                // HBM per particle (the position half of AB is restored from R on demand, ab_positions)
                float4 R0, R1;
                rec32_make(A, un, vn, wn, r, q.eos_any && q.E.on[ar] && q.E.hg[ar], q.E32, (int)t, R0, R1);
                q.R[2 * (size_t)s] = R0;
                q.R[2 * (size_t)s + 1] = R1;
            } else {
                const double m = q.m[g];   // read before the EOS: after it the kernel needs 64 registers, not 62
                float pg, csg;
                if (q.eos_any && q.E.on[ar]) {   // real particle: real_only does not matter here
                    eos_tab_eval(q.E, ar, r, pg, csg);   // the record only: the pool keeps rho
                } else if (eos) {
                    pg = p_eos;
                    csg = cs_eos;
                } else {
                    pg = q.p[g];
                    csg = q.cs[g];
                }
                float4 B, C;
                state_record(un, vn, wn, m, r, pg, csg, (int)t, B, C);
                q.AB[2 * (size_t)s] = A;
                q.AB[2 * (size_t)s + 1] = B;
                q.C[s] = C;
            }
            build_drift(A, q.A0[s], d2, dh);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        d2 = fmaxf(d2, __shfl_xor_sync(0xffffffffu, d2, o));
        dh = fmaxf(dh, __shfl_xor_sync(0xffffffffu, dh, o));
    }
    if (q.reduce_dt) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mc = fmax(mc, __shfl_xor_sync(0xffffffffu, mc, o));
            mf = fmax(mf, __shfl_xor_sync(0xffffffffu, mf, o));
            hm = fmin(hm, __shfl_xor_sync(0xffffffffu, hm, o));
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        s_d2[warp] = d2; s_dh[warp] = dh;
        s_mc[warp] = mc; s_mf[warp] = mf; s_hm[warp] = hm;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < 8; k++) {
            d2 = fmaxf(d2, s_d2[k]); dh = fmaxf(dh, s_dh[k]);
            mc = fmax(mc, s_mc[k]); mf = fmax(mf, s_mf[k]); hm = fmin(hm, s_hm[k]);
        }
        if (d2 > 0.f) atomicMax(&q.red_u32[0], __float_as_uint(d2));
        if (dh > 0.f) atomicMax(&q.red_u32[1], __float_as_uint(dh));
        if (q.reduce_dt) {
            if (mc > -1e299) atomicMax(&q.red[9], d2o(mc));
            if (mf > -1e299) atomicMax(&q.red[11], d2o(mf));
            if (hm < 1e299) atomicMin(&q.red[12], d2o(hm));
        }
    }
}

// 4 CTAs/SM and no spills: at 5 the kernel spilled (36 B) and ran 7 % slower on H100, and with the
// 32-byte records carrying p / rho^2 the spill reloads made it 8 % slower again
__global__ void __launch_bounds__(256, 4) k_stage_pack(const StageArgs a, const FusePackArgs q)
{
    __shared__ float s_d2[8], s_dh[8];
    __shared__ double s_mc[8], s_mf[8], s_hm[8];
    stage_pack_body<false>(a, q, s_d2, s_dh, s_mc, s_mf, s_hm);
}

// k_stage_pack for WCSPHTVDRK3Step (which = 1, 2, 3; dt is used whole): stages 2 and 3 read
// the current state as well as the stage copies.  62 registers, no spills at 4 CTAs/SM.
__global__ void __launch_bounds__(256, 4) k_stage_pack_rk3(const StageArgs a, const FusePackArgs q)
{
    __shared__ float s_d2[8], s_dh[8];
    __shared__ double s_mc[8], s_mf[8], s_hm[8];
    stage_pack_body<true>(a, q, s_d2, s_dh, s_mc, s_mf, s_hm);
}

// What a fused stage 1 with half_pending left unwritten, from the operands that stage read: x .. rho
// = wcsph_combine(x0 .. rho0, f, ax .. arho) with a.au .. a.arho the FIRST evaluation's
// accelerations (the pair pass of the second one writes into the spare set) and the stage's
// factor, and p, cs = the pool side of EP on rho0 (with INIT_RENAMED the stage's rho before the
// EOS calls is rho0).  The same functions on the same doubles: bitwise what the stage would have
// stored.
__global__ void k_half_materialise(const StageArgs a, float *__restrict__ p, float *__restrict__ cs, const int eos_pool,
                                   const EosTab EP)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.pool_end) return;
    const uint8_t t = a.ptype[g];
    if (t == PT_INVALID || (t & PT_GHOST)) return;
    const double f = stage_factor(a.tc, a.f, 1, false);
    a.u[g] = wcsph_combine(a.u0[g], f, a.au[g]);
    a.v[g] = wcsph_combine(a.v0[g], f, a.av[g]);
    a.w[g] = wcsph_combine(a.w0[g], f, a.aw[g]);
    a.x[g] = wcsph_combine(a.x0[g], f, a.ax[g]);
    a.y[g] = wcsph_combine(a.y0[g], f, a.ay[g]);
    a.z[g] = wcsph_combine(a.z0[g], f, a.az[g]);
    a.rho[g] = wcsph_combine(a.rho0[g], f, a.arho[g]);
    if (eos_pool && eos_tab_applies(EP, t)) {
        double rc = a.rho0[g];
        eos_tab_eval(EP, t & 7, rc, p[g], cs[g]);
    }
}

__global__ void k_eos_tab(double *__restrict__ rho, float *__restrict__ p, float *__restrict__ cs,
                          const uint8_t *__restrict__ ptype, long long pool_end, const EosTab E)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= pool_end) return;
    const uint8_t t = ptype[g];
    if (t == PT_INVALID) return;
    eos_tab_apply(rho, p, cs, t, g, E);
}

// R[s] = the 32-byte records (rec32_make) from the packed positions (the position half of AB)
// and the pool's state, with the pending EOS calls applied to the pool on the way (k_eos_tab's
// arithmetic; in the record they only decide the clamp of TaitEOSHGCorrection)
__global__ void k_pack_rec32(const double *__restrict__ u, const double *__restrict__ v,
                             const double *__restrict__ w, double *__restrict__ rho, float *__restrict__ p,
                             float *__restrict__ cs, const uint8_t *__restrict__ ptype,
                             const uint32_t *__restrict__ perm, long long n, const float4 *__restrict__ AB,
                             float4 *__restrict__ R, const EosTab E, const Rec32Eos E32)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = perm[s];
    const uint8_t t = ptype[g];
    eos_tab_apply(rho, p, cs, t, g, E);
    float4 R0, R1;
    rec32_make(AB[2 * s], u[g], v[g], w[g], rho[g], E.on[t & 7] && E.hg[t & 7], E32, (int)t, R0, R1);
    R[2 * s] = R0;
    R[2 * s + 1] = R1;
}

// the position half of AB from the 32-byte records (after k_stage_pack wrote only R):
// the floats pack_position made, for the readers of the 48-byte records
__global__ void k_rec32_positions(const float4 *__restrict__ R, const double *__restrict__ h,
                                  const uint32_t *__restrict__ perm, long long n, float4 *__restrict__ AB)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float4 r = R[2 * s];
    AB[2 * s] = make_float4(r.x, r.y, r.z, (float)h[perm[s]]);
}

// _box_wrap_periodic (nnps_base.pyx:699-743): real and ghost particles alike
__global__ void k_box_wrap(double *__restrict__ x, double *__restrict__ y, double *__restrict__ z,
                           const uint8_t *__restrict__ ptype, long long pool_end, GridDev D /* xmin = lo, cell = L */)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= pool_end || ptype[g] == PT_INVALID) return;
    double *p[3] = {x, y, z};
#pragma unroll
    for (int d = 0; d < 3; d++) {
        if (!D.periodic[d]) continue;
        double v = p[d][g];
        const double lo = D.xmin[d], L = D.cell[d];
        if (v < lo) v += L;
        if (v > lo + L) v -= L;
        p[d][g] = v;
    }
}
__global__ void k_f64_to_f32(const double *__restrict__ in, float *__restrict__ out, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}
__global__ void k_f32_to_f64(const float *__restrict__ in, double *__restrict__ out, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (double)in[i];
}
