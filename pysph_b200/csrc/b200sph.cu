// b200sph.cu -- H100 (sm_90a) evaluator for PySPH's WCSPH per-timestep hot path.
//
// What lives here (see DESIGN.md for the data layout and rooflines):
//   * device mirror of the ParticleArrays: one pool, SoA, fp64 integrated state
//     + fp32 derived fields            (reference: pysph/base/device_helper.py)
//   * NNPS build: bounds/h reductions, cell keys, deterministic counting sort,
//     cell-relative fp32 repack        (reference: pysph/base/nnps_base.pyx:1471-1575,
//                                       linked_list_nnps.pyx:235-382; GPU precedent
//                                       z_order_gpu_nnps_kernels.py:7-47)
//   * fused pair kernel: initialize + loop over all sources + post_loop of
//     SummationDensity / ContinuityEquation / MomentumEquation(+AV) /
//     XSPHCorrection / MonaghanArtificialViscosity
//                                      (reference: acceleration_eval_cython.mako:10-154,
//                                       equation.py:188-297, wc/basic.py:129-269,
//                                       basic_equations.py:19-29,180-300)
//   * TaitEOS / TaitEOSHGCorrection / UpdateSmoothingLengthFerrari, WCSPHStep
//     stages, adaptive-dt reductions   (wc/basic.py:9-126,417-463,
//                                       integrator_step.py:38-91, integrator.py:62-81)
//   * halo pack / append / migrate helpers for the slab decomposition
//                                      (replaces parallel_manager.pyx:512-632)
//
// One translation unit: this file holds the context, the pool and every C-ABI entry
// point; the kernels are included below by family (pool_kernels, scan, nnps_kernels,
// sph_kernels, pair_kernel, pair_list, tvf_kernels, solid_kernels, halo_kernels, density_filter,
// interp_kernels, shift_kernels, iisph_kernels, gtvf_kernels, crksph_kernels .cuh).
//
// No CPU fallback: every entry point needs a CUDA device.
#include "b200sph.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <string>
#include <mutex>
#include <type_traits>
#include <vector>

// --------------------------------------------------------------------------
// small helpers
// --------------------------------------------------------------------------
#define N_PROP_SLOTS (B200SPH_CRK_LAST + 1)   // property ids 0 .. the last CRKSPH property
#define PT_INVALID 0xFFu
#define PT_GHOST 0x08u

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// grid of the grid-stride min / max reductions: 8 blocks of 256 threads on each of an
// H100's 132 SMs
#define REDUCE_BLOCKS (132 * 8)

struct ArrayInfo {
    std::string name;
    int64_t off = 0, cap = 0, n = 0, n_real = 0;
};

struct GridDev {
    double xmin[3];
    double cell[3];   // cell edge per axis (a periodic axis is tiled exactly: L / nc)
    int nc[3];
    int periodic[3];
    int zorder;       // 1: cell ROWS are ordered along the Z-curve of (cy, cz), see grid_row
};

// Cell key = row(cy, cz) * ncx + cx.  x is always the fastest axis, so the 27 neighbour
// cells of a cell are 9 contiguous ranges of the sorted arrays (what the list builder
// streams); the ROWS are ordered row-major (cy + ncy cz) or, zorder, along the Z-curve
// (Morton code) of (cy, cz) -- rows that are close in space are then close in memory
// whatever the aspect ratio of the grid (the reference's GPU NNPS sorts particles by the
// 3-D Morton key of their cell, z_order_nnps.pyx:252-355, z_order.h:24-46).
__host__ __device__ static inline uint32_t part1by1(uint32_t v)
{
    v &= 0x0000ffffu;
    v = (v | (v << 8)) & 0x00ff00ffu;
    v = (v | (v << 4)) & 0x0f0f0f0fu;
    v = (v | (v << 2)) & 0x33333333u;
    v = (v | (v << 1)) & 0x55555555u;
    return v;
}
__host__ __device__ static inline uint32_t compact1by1(uint32_t v)
{
    v &= 0x55555555u;
    v = (v | (v >> 1)) & 0x33333333u;
    v = (v | (v >> 2)) & 0x0f0f0f0fu;
    v = (v | (v >> 4)) & 0x00ff00ffu;
    v = (v | (v >> 8)) & 0x0000ffffu;
    return v;
}
__host__ __device__ static inline uint32_t grid_row(const int zorder, const uint32_t ncy, const uint32_t cy, const uint32_t cz)
{
    return zorder ? (part1by1(cy) | (part1by1(cz) << 1)) : cy + ncy * cz;
}
__host__ __device__ static inline void grid_decode(const int zorder, const uint32_t ncx, const uint32_t ncy, const uint32_t key,
                                                   uint32_t &cx, uint32_t &cy, uint32_t &cz)
{
    cx = key % ncx;
    const uint32_t row = key / ncx;
    if (zorder) {
        cy = compact1by1(row);
        cz = compact1by1(row >> 1);
    } else {
        cy = row % ncy;
        cz = row / ncy;
    }
}

// A = (x, y, z relative to the origin of the cell `key`, h): the packed position of the pair
// records.  ONE function for every writer (the build, the light refresh, the fused stage kernel,
// the ghost refresh), so that they all produce the same floats.
__device__ __forceinline__ float4 pack_position(const GridDev &G, const uint32_t key, const double x, const double y,
                                                const double z, const double h)
{
    uint32_t cx, cy, cz;
    grid_decode(G.zorder, (uint32_t)G.nc[0], (uint32_t)G.nc[1], key, cx, cy, cz);
    float4 a;
    a.x = (float)(x - (G.xmin[0] + (double)cx * G.cell[0]));
    a.y = (float)(y - (G.xmin[1] + (double)cy * G.cell[1]));
    a.z = (float)(z - (G.xmin[2] + (double)cz * G.cell[2]));
    a.w = (float)h;
    return a;
}

// how far the packed position A has drifted from A0, its value at the build:
// d2 = |A - A0|^2, dh = max(h - h_build, 0)
__device__ __forceinline__ void build_drift(const float4 A, const float4 A0, float &d2, float &dh)
{
    const float dx = A.x - A0.x, dy = A.y - A0.y, dz = A.z - A0.z;
    d2 = dx * dx + dy * dy + dz * dz;
    dh = fmaxf(A.w - A0.w, 0.f);
}

// The factor of dt a stage steps by.  With the device-resident dt (tc not null) it is formed
// here from tc[0]: dt / 2 in stage1 of WCSPHStep (and of EDACStep, EDACTVFStep, SolidMechStep),
// dt in their stage2 and in every stage of WCSPHTVDRK3Step (whole); otherwise it is the host's
// factor f.  Every stage kernel, fused or not, takes its factor from here.
__device__ __forceinline__ double stage_factor(const double *tc, const double f, const int which, const bool whole)
{
    if (!tc) return f;
    const double dt = tc[0];
    return whole || which != 1 ? dt : 0.5 * dt;
}

// equation-of-state calls wait here until the next k_pack_state applies them in the
// same pass that gathers the state into the pair records (saves one launch and one
// sweep over rho/p/cs per array and evaluation); eos_flush() runs them stand-alone
// if something reads rho/p/cs before that.
struct EosTab {
    int on[B200SPH_MAX_ARRAYS], hg[B200SPH_MAX_ARRAYS], real_only[B200SPH_MAX_ARRAYS];
    double rho0[B200SPH_MAX_ARRAYS], c0[B200SPH_MAX_ARRAYS], gamma[B200SPH_MAX_ARRAYS], p0[B200SPH_MAX_ARRAYS];
};

// ratio^gamma and ratio^((gamma - 1) / 2) of the Tait equation of state (wc/basic.py:60-65,
// :118-126).  Water's gamma = 7 -- every WCSPH example of the reference -- needs no pow():
// five fp64 multiplications, within 3 ulp of pow() (the results are stored as fp32); any
// other exponent takes the library route.  ONE function for every kernel that evaluates
// the EOS, so that they all produce the same bits.
__host__ __device__ static inline void tait_powers(const double ratio, const double gamma, double &rg, double &rh)
{
    if (gamma == 7.0) {
        const double r2 = ratio * ratio;
        rh = r2 * ratio;
        rg = rh * rh * ratio;
    } else {
        rg = pow(ratio, gamma);
        rh = pow(ratio, 0.5 * (gamma - 1.0));
    }
}

// TaitEOS.loop wc/basic.py:60-65 ; TaitEOSHGCorrection.loop wc/basic.py:118-126 on one particle
// of array a: the rho clamp of the HG variant (r clamped in place; true when it was), p and cs.
// The one evaluation of the EOS: every kernel that applies it calls this, and decides itself
// whether the clamped rho goes back to the pool or stays in its record.
__device__ __forceinline__ bool eos_tab_applies(const EosTab &E, const uint8_t t)
{
    const int a = t & 7;
    return E.on[a] && !(E.real_only[a] && (t & PT_GHOST));
}
__device__ __forceinline__ bool eos_tab_eval(const EosTab &E, const int a, double &r, float &p, float &cs)
{
    const double rho0 = E.rho0[a];
    const bool clamp = E.hg[a] && r < rho0;
    if (clamp) r = rho0;
    const double ratio = r * (1.0 / rho0);
    const double Bc = rho0 * E.c0[a] * E.c0[a] / E.gamma[a];
    double rg, rh;
    tait_powers(ratio, E.gamma[a], rg, rh);
    p = (float)((E.hg[a] ? 0.0 : E.p0[a]) + Bc * (rg - 1.0));
    cs = (float)(E.c0[a] * rh);
    return clamp;
}

// B = (u, v, w, m), C = (rho, p / rho^2, cs, type): the state half of the 48-byte pair records.
// ONE function for every writer, so that they all produce the same floats.
__device__ __forceinline__ void state_record(const double u, const double v, const double w, const double m, const double r,
                                             const float p, const float cs, const int t, float4 &B, float4 &C)
{
    B.x = (float)u; B.y = (float)v; B.z = (float)w; B.w = (float)m;
    C.x = (float)r;
    C.y = (float)((double)p / (r * r));
    C.z = cs;
    C.w = __int_as_float(t);
}

// The one Tait EOS (gamma = 7) the 32-byte records are formed with: rho0, B = rho0 c0^2 / 7 and
// the pressure offset (p0 of TaitEOS, 0 with TaitEOSHGCorrection).  The records depend on these
// three values only, so they are also the key that says when the records must be repacked.
struct Rec32Eos {
    double rho0, B, poff;
    // folded on the host for rec32_make: kB (1, 7, 21, 35) with kB = B / rho0^2, and poff / rho0^2
    float tait[4], kp;
    bool operator!=(const Rec32Eos &o) const { return rho0 != o.rho0 || B != o.B || poff != o.poff; }
};

struct PendingEvent {
    cudaEvent_t e0, e1;
    int slot;  // 0 nnps, 1 pair, 2 other
};

// A buffer the context owns: `cap` elements of device memory, or of page-locked host memory
// (PINNED: cudaMallocHost; MAPPED: cudaHostAlloc with a device alias).  It frees itself, so the
// context frees every buffer by being deleted; grow() below is the one place that allocates.
// It reads as the raw pointer (launches, argument structs, copies).
enum class Mem { DEVICE, PINNED, MAPPED };
template <class T, Mem M = Mem::DEVICE> struct Buf {
    T *p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(Buf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; }
    Buf &operator=(Buf &&o) noexcept { std::swap(p, o.p), std::swap(cap, o.cap); return *this; }
    ~Buf() { reset(); }
    cudaError_t reset()
    {
        const cudaError_t e = !p ? cudaSuccess : M == Mem::DEVICE ? cudaFree(p) : cudaFreeHost(p);
        p = nullptr, cap = 0;
        return e;
    }
    operator T *() const { return p; }
    T *operator->() const { return p; }
};
struct PeerBox;
struct PeerDecision;
struct ShiftRec;    // shift_kernels.cuh
struct IisphState;  // iisph_kernels.cuh

struct b200sph_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;            // last error of the calling threads' entry points ...
    std::string err_out;        // ... and the copy b200sph_last_error hands out
    std::mutex err_mu;          // the output thread (snapshot_fetch / release) reports errors too

    int narr = 0;
    ArrayInfo arr[B200SPH_MAX_ARRAYS];
    int64_t pool_cap = 0;   // allocated particles in the pool
    int64_t pool_end = 0;   // off[last] + cap[last]
    // the property buffers by property id (prop_kind: element type and when it is allocated; null
    // until then, and for ids the header does not define).  Which buffer goes by x .. rho and
    // which by x0 .. rho0 changes when a fused stage 1 takes the initialize by renaming
    // (init_by_rename): read these at enqueue time, and keep no copy of them across a stage
    void *prop[N_PROP_SLOTS] = {nullptr};
    Buf<float4> Dv;                     // sorted: (uhat-u, vhat-v, what-w, pavg)
    Buf<float4> T01, T2R, R2;           // sorted stress records (with the elastic group)
    Buf<float2> PT;                     // sorted: (p, type)
    Buf<uint8_t> ptype;
    bool ptype_dirty = true;

    int kernel = 0, dim = 3;
    double radius_scale = 2.0;

    // domain manager
    bool periodic[3] = {false, false, false};
    double dom_lo[3] = {0, 0, 0}, dom_hi[3] = {0, 0, 0};
    // mirror boundaries (b200sph_set_mirror): images are materialised as tag=Ghost particles
    bool mirror[3] = {false, false, false};
    double mirror_layers = 2.0;
    struct MirrorSeg {
        int arr, axis, side;
        int64_t count = 0, ghost_first = 0;             // ghost_first: relative to the array's first ghost
        Buf<uint32_t> idx;                              // sources, relative to the array's offset
    };
    std::vector<MirrorSeg> mirror_segs;                 // in creation order (corner images read earlier ones)
    bool mirror_built = false;
    double cell_size = 1.0, hmin_scaled = 1.0;
    bool domain_valid = false;
    // grid
    b200sph_grid_info grid;
    bool grid_valid = false;
    bool packed_valid = false;  // A / AB hold the CURRENT positions (set by a light update, the fused stage kernel or peer_begin; kept by peer_recv)
    double last_domain_size = 0.0;

    // sort / cell list buffers
    Buf<uint32_t> key_of;        // [pool] cell key per particle
    Buf<uint32_t> off_in;        // [pool] arrival rank inside the cell
    Buf<uint32_t> cell_cnt, cell_start;
    Buf<uint32_t> blk_sums;
    Buf<uint32_t> perm_tmp, perm, skey, rank;
    Buf<float4> A, B, C;
    Buf<float4> AB;  // {A, B} interleaved (32 B = one sector per particle) for the list consumer's 256-bit gathers
    // the 32-byte records of the WCSPH pass (records32): {(x, y, z, p / rho^2), (u, v, w, delta + type)};
    // while rec32 holds, the state records are packed HERE instead of B / C / the B half of AB
    Buf<float4> R;
    bool rec32 = false;
    Rec32Eos rec32_eos = {};    // the EOS the records are packed with
    bool ab_stale = false;      // k_stage_pack wrote the positions into R only (ab_positions restores AB)
    bool rec48_forced = false;  // env B200SPH_RECORDS=48
    // h and m over all particles (records32 needs both uniform): computed on demand by one
    // min/max reduction, cleared by set_changed / h_changed / m_changed
    bool hm_known = false;
    double h_uniform = NAN, m_uniform = NAN;   // NaN: not uniform
    int64_t n_pair_r32 = 0;
    int64_t n_sorted = 0;
    bool state_packed = false;
    int force_kernel = 0;       // 0 lists (default), 1 warp kernel (env B200SPH_PAIR_KERNEL)
    bool zorder = false;        // cell rows along the Z-curve of (cy, cz) (env B200SPH_ZORDER)
    // persistent neighbour lists
    double skin = 0.1;          // S = skin * radius_scale * hmax, adapted between skin_min and skin_max
    double skin_max = 0.1;      // env B200SPH_SKIN (also what a halo exchange must cover)
    double skin_min = 0.02;
    bool skin_adapt = true;     // env B200SPH_SKIN_ADAPT=0 switches the controller off
    int64_t evals_since_build = 0;  // light updates served by the current build
    double skin_next = -1.0;        // set by retire_build: the skin of the next build (else the geometric rule)
    double S_abs = 0.0;         // absolute skin of the current build
    double cell_int = 1.0;      // internal cell size (cell_size + S)
    GridDev G;                  // frozen device grid of the current build
    Buf<float4> A0;             // packed positions at build time
    Buf<uint32_t> lst;          // transposed lists: [n/32][capg][32]
    Buf<uint32_t> cnt;          // [n] list length per destination
    int capg = 0;               // entries reserved per destination
    bool lists_valid = false;
    bool topo_dirty = true;     // particle set / h pushed: a light update is not enough
    bool drift_ok = false;      // set by nnps_drift when its caller took the (collective) decision
    // deferred drift check (b200sph_nnps_update_deferred / b200sph_nnps_confirm)
    bool defer_check = false;   // the running nnps_update may leave its drift check pending
    bool check_pending = false; // a light update ran on the assumption that the lists are valid
    Buf<unsigned, Mem::PINNED> drift_host;
    cudaEvent_t drift_evt = nullptr;
    int64_t n_deferred_failed = 0;
    // proactive rebuild: the used-up fraction of the skin at the last two confirmed deferred
    // checks of the current build; when their extrapolation says the NEXT evaluation would
    // fail its check, the lists are rebuilt before it instead of after a wasted evaluation
    double drift_hist[2] = {-1.0, -1.0};
    bool proactive = true;      // env B200SPH_PROACTIVE=0
    int64_t n_proactive = 0;
    // device-resident time control block: [0] dt, [1] t, [2] proposed dt, [3] h_minimum
    double *tc = nullptr;               // tc_own, or the caller's block (b200sph_time_control)
    Buf<double> tc_own;
    Buf<double, Mem::PINNED> tc_host;   // 2 snapshot slots x 2 doubles
    double t_final = INFINITY, t_eps = 0.0;  // b200sph_time_final: the last dt lands on t_final
    // asynchronous output snapshot (b200sph_snapshot_*): one in flight
    Buf<double> snap_buf;               // device staging, 8-byte slots
    std::vector<int64_t> snap_off, snap_len;   // per segment: offset (doubles) / elements
    std::vector<int> snap_u32;          // per segment: 1 = 4-byte integers
    cudaStream_t snap_stream = nullptr; // the D2H copies run here, beside the time loop
    cudaEvent_t snap_ready = nullptr, snap_done = nullptr;
    std::atomic<bool> snap_open{false};   // taken by the time loop, released by the output thread
    cudaEvent_t tc_evt[2] = {nullptr, nullptr};
    bool h_dirty = true;        // h changed since the last update_domain reduction
    Buf<unsigned> red_u32;
    Buf<unsigned, Mem::PINNED> red_u32_host;
    int64_t n_full_builds = 0, n_light_updates = 0, n_list_builds = 0;

    // scratch
    Buf<long long> red;           // 16 ordered-int64 slots
    Buf<long long, Mem::PINNED> red_host;
    Buf<unsigned long long> counter;  // pair counter + misc
    Buf<unsigned long long, Mem::PINNED> counter_host;
    Buf<double> stage_buf;        // host<->device staging for f32 props
    Buf<uint32_t> flag_a, flag_b; // [pool+1] scan scratch

    // persistent halo: pool-relative indices of the real particles sent to neighbour `slot`
    Buf<uint32_t> halo_idx[B200SPH_MAX_ARRAYS][2];
    int64_t halo_cnt[B200SPH_MAX_ARRAYS][2] = {{0}};

    EosTab eos_pending;
    bool eos_any = false;
    // the pool side (rho clamp, p, cs) of EOS calls a pair pass has already put into the records,
    // left for the next fused stage kernel; eos_flush runs it stand-alone (before eos_pending)
    EosTab eos_pool;
    bool eos_pool_any = false;
    // ---- peer protocol (b200sph_peer_*) + interior / boundary split of the list consumer --
    int peer_rank = -1, peer_world = 0;
    Buf<PeerBox> peer_box;                       // this rank's mailbox
    PeerBox *peer_boxes[B200SPH_MAX_RANKS] = {nullptr};   // every rank's (own: the local one)
    bool peer_connected = false;
    unsigned long long peer_epoch = 0, peer_dt_epoch = 0;
    Buf<unsigned> peer_done;                     // "blocks finished" counters of k_peer_push, one per direction
    Buf<double> peer_dec_dev;
    Buf<PeerDecision, Mem::MAPPED> peer_dec_host;
    PeerDecision *peer_dec_hostdev = nullptr;    // the device alias of peer_dec_host
    cudaStream_t comm_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // profiling of the overlapped evaluation (b200sph_set_profiling != 0): per pair pass an event
    // triple {fork of the communication stream, scatter done, boundary launch done}
    struct HaloEvents { cudaEvent_t fork, chain, end, sent, reduced; };
    std::vector<HaloEvents> halo_pending;
    cudaEvent_t halo_ev_fork = nullptr, halo_ev_chain = nullptr, halo_ev_sent = nullptr, halo_ev_reduced = nullptr;
    bool comm_pending = false;                   // work on comm_stream that the main stream has not waited for
    // The scalar agreement runs on its own stream: a rank's ghosts only need its two neighbours,
    // the decision needs every rank, and the boundary launch must not wait for the slowest one.
    cudaStream_t red_stream = nullptr;
    // generic-equation fallback: run-time compiled modules
    std::vector<void *> gen_modules;             // CUmodule (or, emulated, a dlopen handle)
    // density_filter: its records, [2 n_sorted] (allocated on first use)
    Buf<float4> dfilter_F;
    // interpolation (b200sph_probe_*, b200sph_interpolate): the probe sets by id (xyz: 3 n doubles,
    // null once released), the records [2 n_sorted] and order1's rho [n_sorted], the reach
    // reduction and the results (allocated on first use)
    struct ProbeSet { Buf<double> xyz; int64_t n = 0; double h = 0.0; };
    std::vector<ProbeSet> probes;
    Buf<float4> interp_Q;
    Buf<float> interp_rho;
    Buf<unsigned> interp_red;
    Buf<double> interp_out;
    // particle shifting (b200sph_shift, b200sph_correct_velocities): the fp64 records [n_sorted]
    // each, dpos and the velocity change [3 pool_end] by gid, max |v| per array; shift_mask: the
    // arrays whose dpos is in shift_dpos
    Buf<ShiftRec> shift_P, shift_V;
    Buf<double> shift_dpos, shift_dvel;
    Buf<long long> shift_vmax;
    unsigned shift_mask = 0;
    // implicit incompressible SPH (b200sph_iisph_pass): the position records [n_sorted], the new
    // pressure of an iteration [pool_end], the partial sums of its reduction and the iteration
    // state.  iisph_spec: an IISPH evaluation ran on a deferred drift check not yet confirmed;
    // iisph_restore: that check failed, so the repeat starts from p = p0 (the step's pressure)
    Buf<ShiftRec> iisph_P;
    Buf<double> iisph_pnext, iisph_part;
    Buf<IisphState> iisph_st;
    bool iisph_spec = false, iisph_restore = false;
    // the generalised transport-velocity formulation (b200sph_gtvf_pass): the position records
    // [n_sorted].  gtvf_spec: an evaluation 1 ran on a deferred drift check not yet confirmed;
    // gtvf_restore: that check failed, so the repeat keeps rho0 (the density of stage 2)
    Buf<ShiftRec> gtvf_P;
    // conservative reproducing-kernel SPH (b200sph_crksph_pass): the position records [n_sorted]
    Buf<ShiftRec> crk_P;
    bool gtvf_spec = false, gtvf_restore = false;
    // Group(start_idx, stop_idx): one-shot destination ranges of the next pair pass
    int64_t dst_lo[B200SPH_MAX_ARRAYS] = {0}, dst_hi[B200SPH_MAX_ARRAYS] = {0};
    bool dst_ranged = false;
    cudaEvent_t ev_pushed = nullptr, ev_red = nullptr;
    // peer_publish / peer_send / peer_recv only RECORD: the launches are merged into one
    // k_peer_push (at peer_reduce) and one k_peer_pull (at peer_end)
    struct PeerPending *pend = nullptr;
    Buf<uint8_t> sflag;                          // [sorted] 1 = ghost
    Buf<uint8_t> stype;                          // [sorted] particle type byte (array id | ghost bit), written by k_pack_pos
    unsigned long long list_mask[B200SPH_MAX_ARRAYS] = {0};   // the equation mask the current lists were filtered with
    Buf<uint32_t> chunk_boundary, chunk_interior;
    int64_t n_chunk_boundary = 0, n_chunk_interior = 0;
    bool chunks_valid = false;
    int64_t n_overlapped = 0;
    // ---- fused stage kernel (k_stage_pack) bookkeeping ---------------------------------
    bool fuse = true;            // env B200SPH_FUSE=0: the unfused kernels only
    EosTab eos_last;             // the equation-of-state calls of the last evaluation ...
    bool eos_last_valid = false;
    bool spec_records = false;   // ... were applied to the packed records speculatively
    unsigned spec_confirmed = 0; // arrays whose b200sph_eos call has matched the speculation
    bool drift_measured = false; // red_u32 holds the drift of the CURRENT packed positions
    bool red_armed = false;      // red[9,11,12] hold their neutral values
    bool dt_reduced = false;     // ... hold the factors of the last evaluation (fused stage2)
    bool dt_adaptive_seen = false;  // a dt proposal followed the last stage2: reduce in the next one
    bool init_pending = false;   // an initialize of every array waits for the next fused stage (init_materialise)
    int64_t n_fused = 0;
    // a fused WCSPHStep stage 1 left x .. rho and the pool side of its EOS calls unwritten
    // (half_materialise forms them from what the stage read: its factor, its EOS calls)
    bool half_pending = false;
    double half_f = 0.0;
    const double *half_tc = nullptr;
    int half_eos = 0;
    EosTab half_EP;
    int64_t n_half_materialised = 0;
    // the second set of arho, au .. az (acc_swap); acc_swapped: the pair pass after that stage 1 writes
    // into it, and acc_spare holds the accelerations the stage read.  acc_differ: where the two
    // sets may hold different values (ACC_* bits); the pair passes do not write every array's
    // accelerations, and the ones they leave must be the same in both sets
    Buf<float> acc_spare[7];   // arho, au .. az: the property ids B200SPH_ARHO .. B200SPH_AZ
    bool acc_swapped = false;
    unsigned acc_differ = ~0u;

    // stats
    b200sph_stats stats;
    int profiling = 0;          // 0 off, 1 every phase, 2 the pair kernels only
    bool async_copies = false;  // push/pull return without waiting (pinned host buffers)
    std::vector<PendingEvent> pending;
    std::vector<cudaEvent_t> ev_pool;
};

// ---- what a change invalidates ----------------------------------------------------------
// The flags above cache work that later calls reuse.  An entry point that changes the
// particles calls one of these transitions; a flag becomes valid again only where its work
// is done (the full build, build_lists, pack_state, k_stage_pack, the drift checks and the
// ghost repacks).

// Positions or h of the same particles changed: the grid and the packed positions are stale.
// The build may survive: nnps_update measures the drift against it.  The 32-byte records
// carry the positions as well: only k_stage_pack rewrites them with the positions (and says
// so); the next nnps_update rewrites the position half of AB, unless k_stage_pack did (then
// it sets ab_stale again).
static void positions_changed(b200sph_ctx *ctx)
{
    ctx->grid_valid = false, ctx->packed_valid = false;
    if (ctx->rec32) ctx->state_packed = false;
    ctx->ab_stale = false;
}

// A property the pair records (B, C) are made of changed, or B / C now hold other records:
// the next pair pass packs them again.
static void state_changed(b200sph_ctx *ctx) { ctx->state_packed = false; }

// The same particles moved and changed state (a stage, a ghost refresh, a periodic wrap).
static void particles_moved(b200sph_ctx *ctx)
{
    positions_changed(ctx);
    state_changed(ctx);
}

// h changed: the packed positions carry it, and update_domain must reduce hmin / hmax again.
static void h_changed(b200sph_ctx *ctx)
{
    positions_changed(ctx);
    ctx->domain_valid = false, ctx->h_dirty = true;
    ctx->hm_known = false;
}

// m changed (a push, or a generic Group that stores to the state): records32 must look at
// the masses again.
static void m_changed(b200sph_ctx *ctx) { ctx->hm_known = false; }

// The build cannot be reused (domain, mirror planes or kernel support changed, or a deferred
// drift check failed): the next nnps_update makes a full build, which repacks the state.
// state_packed needs no clearing here: every reader of it needs grid_valid or a reusable
// build, and neither returns before that full build.
static void build_invalid(b200sph_ctx *ctx)
{
    positions_changed(ctx);
    ctx->topo_dirty = true;
}

// The particle set changed: the build, the type table and the h reduction are stale.  The
// last hmin / hmax stay in use by nnps_update until update_domain runs: after add_array /
// resize_array the caller pushes the new values (push_f64 of h invalidates them), after
// drop_ghosts the halo appends the new ghosts.
static void set_changed(b200sph_ctx *ctx)
{
    build_invalid(ctx);
    state_changed(ctx);
    ctx->ptype_dirty = true, ctx->h_dirty = true;
    ctx->hm_known = false;
    ctx->shift_mask = 0;   // the gids of the last shift's dpos may name other particles now
}

// Particles arrived or left with their own h (halo_append, migrate_out, mirror images): the
// next nnps_update reduces h again before it builds.
static void set_changed_with_h(b200sph_ctx *ctx)
{
    set_changed(ctx);
    ctx->domain_valid = false;
}

// The pool was laid out anew and every sorted buffer reallocated: the lists are gone as well
// (and the skin controller must not judge the lifetime of a build that did not end by drift).
static void pool_moved(b200sph_ctx *ctx)
{
    set_changed(ctx);
    ctx->lists_valid = false;
}

// Ghost values were overwritten in place (peer_recv).  With a reusable
// build whose packed positions are current, the same launch repacks the ghosts' positions
// (`repacked`) and, `records`, their state records: those flags stay.
static void ghosts_refreshed(b200sph_ctx *ctx, bool repacked, bool records)
{
    ctx->grid_valid = false;
    if (!repacked) ctx->packed_valid = false;
    if (!records) state_changed(ctx);
}

// The lists no longer serve (they do not cover what a pass needs, or a new build replaces
// them); the ghost-free chunks were derived from them.
static void lists_stale(b200sph_ctx *ctx) { ctx->lists_valid = false, ctx->chunks_valid = false; }

// A light update has judged the drift measured with the packed positions: the next check
// measures again.
static void drift_consumed(b200sph_ctx *ctx) { ctx->drift_measured = false; }

struct PhaseTimer;
static int set_err(b200sph_ctx *c, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) {
        std::lock_guard<std::mutex> lk(c->err_mu);
        c->err = buf;
    }
    return -1;
}

#define CU(call)                                                                    \
    do {                                                                            \
        cudaError_t _e = (call);                                                    \
        if (_e != cudaSuccess)                                                      \
            return set_err(ctx, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                     \
    } while (0)

// b holds at least `need` elements afterwards: a smaller buffer is freed and `reserve` (>= need)
// elements are allocated -- freed first, so that the old and the new one never take the card
// together.  Contents are not kept.  On failure b is left empty.
template <class T, Mem M> static int grow(b200sph_ctx *ctx, Buf<T, M> &b, size_t need, size_t reserve)
{
    if (need <= b.cap) return 0;
    cudaError_t e = b.reset();
    const size_t bytes = sizeof(T) * reserve;
    if (e == cudaSuccess)
        e = M == Mem::DEVICE ? cudaMalloc((void **)&b.p, bytes)
          : M == Mem::PINNED ? cudaMallocHost((void **)&b.p, bytes)
                             : cudaHostAlloc((void **)&b.p, bytes, cudaHostAllocMapped);
    if (e != cudaSuccess) {
        b.p = nullptr;
        return set_err(ctx, "cannot allocate %.1f MB of %s memory: %s", 1e-6 * (double)bytes,
                       M == Mem::DEVICE ? "device" : "pinned host", cudaGetErrorString(e));
    }
    b.cap = reserve;
    return 0;
}

#define LAUNCH_CHECK()                                                              \
    do {                                                                            \
        ctx->stats.kernel_launches++;                                               \
        cudaError_t _e = cudaGetLastError();                                        \
        if (_e != cudaSuccess)                                                      \
            return set_err(ctx, "kernel launch failed: %s (%s:%d)",                 \
                           cudaGetErrorString(_e), __FILE__, __LINE__);             \
    } while (0)

// ordered-int64 image of a double so atomicMin/Max(long long) order like doubles
__host__ __device__ static inline long long d2o(double d)
{
    long long b;
#ifdef __CUDA_ARCH__
    b = __double_as_longlong(d);
#else
    memcpy(&b, &d, 8);
#endif
    return b ^ ((b >> 63) & 0x7fffffffffffffffLL);
}
__host__ __device__ static inline double o2d(long long o)
{
    long long b = o ^ ((o >> 63) & 0x7fffffffffffffffLL);
#ifdef __CUDA_ARCH__
    return __longlong_as_double(b);
#else
    double d;
    memcpy(&d, &b, 8);
    return d;
#endif
}

__device__ __forceinline__ float frcp(float x)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float frsqrt(float x)
{
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// nanosecond clock shared by every SM (bounds the spin waits of the peer protocol); the
// host emulation of the tests supplies its own
#ifndef B200SPH_HOST_EMULATION
__device__ __forceinline__ unsigned long long peer_now_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#endif

#include "generic_args.h"
// The 32-byte record of the WCSPH pass when h, m and the Tait EOS (gamma = 7) are the same for
// every particle (records32 in b200sph.cu): R = {(x, y, z, tau), (u, v, w, delta')} with
//   delta = rho / rho0 - 1 formed in fp64 after the clamp of TaitEOSHGCorrection, so that fp32
//     keeps the digits of the density variation;
//   tau = p / rho^2 = (kB ((1 + delta)^7 - 1) + kp) / (1 + delta)^2, the source's pressure term,
//     from delta in fp32 (the Tait polynomial in Horner form: no cancellation for small delta)
//     -- the arithmetic k_pair_list_r32 used to repeat for every pair, so the same bits;
//   delta' = delta with the array type (0..7; no ghosts on this path) in its 3 low mantissa bits.
//     That moves delta by at most 7 ulp, ~1e-9 rho0 at |delta| <= 0.02, far below the fp32
//     rounding of rho; k_pair_list_r32 takes rho and cs from delta' as it is, the type from its
//     low bits.
// ONE function for every writer, so that they all produce the same bits.
__device__ __forceinline__ void rec32_make(const float4 A, const double u, const double v, const double w, double rho,
                                           const bool clamp, const Rec32Eos &E, const int type, float4 &R0, float4 &R1)
{
    if (clamp && rho < E.rho0) rho = E.rho0;
    const float d = (float)(rho * (1.0 / E.rho0) - 1.0);
    const float x = 1.0f + d;
    const float t = fmaf(fmaf(fmaf(fmaf(fmaf(d, E.tait[0], E.tait[1]), d, E.tait[2]), d, E.tait[3]), d, E.tait[3]), d, E.tait[2]);
    R0 = make_float4(A.x, A.y, A.z, fmaf(fmaf(t, d, E.tait[1]), d, E.kp) * frcp(x * x));
    R1 = make_float4((float)u, (float)v, (float)w, __int_as_float((__float_as_int(d) & ~7) | (type & 7)));
}

#include "pool_kernels.cuh"
#include "scan.cuh"
#include "nnps_kernels.cuh"
#include "sph_kernels.cuh"
#include "pair_kernel.cuh"
#include "pair_list.cuh"
#include "tvf_kernels.cuh"
#include "solid_kernels.cuh"
#include "halo_kernels.cuh"
#include "density_filter.cuh"
#include "interp_kernels.cuh"
#include "shift_kernels.cuh"
#include "iisph_kernels.cuh"
#include "gtvf_kernels.cuh"
#include "crksph_kernels.cuh"

// --------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------
// What a property id of the header's enum is: its element type on the device (PROP_NONE: no such
// property) and when its buffer is allocated -- with the pool, as a group the first time any
// elastic-dynamics property is named (with the stress records T01 T2R R2), as a group the first
// time any IISPH property is named, or one by one when a
// user property is named.  The only host code that knows the ranges of the id enum.
enum PropType { PROP_NONE, PROP_F64, PROP_F32, PROP_U32 };
enum PropGroup { GROUP_POOL, GROUP_ELASTIC, GROUP_IISPH, GROUP_GTVF, GROUP_CRKSPH, GROUP_USER };
struct PropKind {
    PropType type;
    PropGroup group;
    size_t size() const { return type == PROP_F64 ? 8 : 4; }
};
static PropKind prop_kind(int p)
{
    if (p >= B200SPH_X && p <= B200SPH_RHO0) return {PROP_F64, GROUP_POOL};
    if (p >= B200SPH_P && p <= B200SPH_DT_FORCE) return {PROP_F32, GROUP_POOL};
    if (p >= B200SPH_UHAT && p <= B200SPH_PF0) return {PROP_F64, GROUP_POOL};
    if (p >= B200SPH_VOL && p <= B200SPH_AP) return {PROP_F32, GROUP_POOL};
    if (p >= B200SPH_GID && p <= B200SPH_PID) return {PROP_U32, GROUP_POOL};
    if (p >= B200SPH_S00 && p <= B200SPH_S220) return {PROP_F64, GROUP_ELASTIC};
    if (p >= B200SPH_V00 && p <= B200SPH_AS22) return {PROP_F32, GROUP_ELASTIC};
    if (p >= B200SPH_UADV && p <= B200SPH_IISPH_V) return {PROP_F64, GROUP_IISPH};
    if (p >= B200SPH_RHODIV && p <= B200SPH_GTVF_P0) return {PROP_F64, GROUP_GTVF};
    if (p >= B200SPH_CRK_E && p <= B200SPH_CRK_LAST) return {PROP_F64, GROUP_CRKSPH};
    if (p >= B200SPH_USER0 && p < B200SPH_USER0 + B200SPH_MAX_USER) return {PROP_F64, GROUP_USER};
    return {PROP_NONE, GROUP_POOL};
}
static double *f64_ptr(const b200sph_ctx *ctx, int p) { return (double *)ctx->prop[p]; }
static float *f32_ptr(const b200sph_ctx *ctx, int p) { return (float *)ctx->prop[p]; }
static uint32_t *u32_ptr(const b200sph_ctx *ctx, int p) { return (uint32_t *)ctx->prop[p]; }
static bool elastic_allocated(const b200sph_ctx *ctx) { return ctx->prop[B200SPH_S00] != nullptr; }

// the neighbour lists can index n particles (26-bit sorted indices; beyond, and with
// B200SPH_PAIR_KERNEL=warp, the list-free kernel runs)
static bool lists_usable(const b200sph_ctx *ctx, int64_t n) { return ctx->force_kernel == 0 && n < (1LL << LIST_JBITS); }
// the current build's sorted order and lists can serve a light update
static bool reusable_build(const b200sph_ctx *ctx) { return ctx->force_kernel == 0 && ctx->lists_valid && !ctx->topo_dirty; }
// the fused stage `which` (it steps every array) may take a pending initialize by exchanging
// the buffers x .. rho and x0 .. rho0 instead of copying one into the other: the stepped state
// then exists in the new x .. rho only where this launch writes it, so every particle must be
// one it steps -- no ghosts -- and it must not read the current state beside the stage copies,
// which TVD-RK3's stages 2 and 3 do
static bool init_by_rename(const b200sph_ctx *ctx, int which)
{
    if (which != 1) return false;
    for (int a = 0; a < ctx->narr; a++)
        if (ctx->arr[a].n != ctx->arr[a].n_real) return false;
    return true;
}

// (re)build the pool so that every array owns [off, off+cap); moves existing data.
static int pool_layout(b200sph_ctx *ctx, const int64_t *new_cap)
{
    int64_t new_off[B200SPH_MAX_ARRAYS], total = 0;
    for (int a = 0; a < ctx->narr; a++) {
        new_off[a] = total;
        total += (new_cap[a] + 31) / 32 * 32;
    }
    const int64_t alloc = std::max<int64_t>(total, 32);
    // allocate new buffers and move array by array: the pool's properties and those of the
    // other groups that are allocated
    for (int p = 0; p < N_PROP_SLOTS; p++) {
        const PropKind pk = prop_kind(p);
        if (pk.type == PROP_NONE || (pk.group != GROUP_POOL && !ctx->prop[p])) continue;
        const size_t esz = pk.size();
        void *old = ctx->prop[p];
        void *nw = nullptr;
        CU(cudaMalloc(&nw, esz * (size_t)alloc));
        CU(cudaMemsetAsync(nw, 0, esz * (size_t)alloc, ctx->stream));
        if (old) {
            for (int a = 0; a < ctx->narr; a++) {
                if (ctx->arr[a].n > 0 && ctx->arr[a].cap > 0)
                    CU(cudaMemcpyAsync((char *)nw + esz * (size_t)new_off[a],
                                       (char *)old + esz * (size_t)ctx->arr[a].off,
                                       esz * (size_t)ctx->arr[a].n, cudaMemcpyDeviceToDevice,
                                       ctx->stream));
            }
            CU(cudaStreamSynchronize(ctx->stream));
            CU(cudaFree(old));
        }
        ctx->prop[p] = nw;
    }
    for (int a = 0; a < ctx->narr; a++) {
        ctx->arr[a].off = new_off[a];
        ctx->arr[a].cap = new_cap[a];
    }
    ctx->pool_cap = alloc;
    ctx->pool_end = total;
    pool_moved(ctx);
    // per-particle work buffers (their contents are stale now): AB and R hold two float4 per
    // particle, the scan scratch flag_a / flag_b one entry more
    const size_t n = (size_t)alloc;
    int rc;
    for (Buf<uint32_t> *b : {&ctx->key_of, &ctx->off_in, &ctx->perm_tmp, &ctx->perm, &ctx->skey, &ctx->rank, &ctx->cnt})
        if ((rc = grow(ctx, *b, n, n))) return rc;
    for (Buf<uint32_t> *b : {&ctx->flag_a, &ctx->flag_b})
        if ((rc = grow(ctx, *b, n + 1, n + 1))) return rc;
    for (Buf<float4> *b : {&ctx->A, &ctx->B, &ctx->C, &ctx->A0, &ctx->Dv})
        if ((rc = grow(ctx, *b, n, n))) return rc;
    for (Buf<float4> *b : {&ctx->AB, &ctx->R})
        if ((rc = grow(ctx, *b, 2 * n, 2 * n))) return rc;
    for (Buf<uint8_t> *b : {&ctx->ptype, &ctx->stype})
        if ((rc = grow(ctx, *b, n, n))) return rc;
    if ((rc = grow(ctx, ctx->PT, n, n))) return rc;
    if (elastic_allocated(ctx))
        for (Buf<float4> *b : {&ctx->T01, &ctx->T2R, &ctx->R2})
            if ((rc = grow(ctx, *b, n, n))) return rc;
    for (Buf<float> &b : ctx->acc_spare) CU(b.reset());   // (acc_swap allocates it again, at pool_cap)
    ctx->acc_differ = ~0u;
    return 0;
}

static int ensure_capacity(b200sph_ctx *ctx, int arr, int64_t need)
{
    if (need <= ctx->arr[arr].cap && ctx->pool_cap > 0) return 0;
    int64_t caps[B200SPH_MAX_ARRAYS];
    for (int a = 0; a < ctx->narr; a++) caps[a] = ctx->arr[a].cap;
    if (need > caps[arr]) caps[arr] = need + need / 4 + 1024;
    return pool_layout(ctx, caps);
}

static int refresh_ptype(b200sph_ctx *ctx)
{
    if (!ctx->ptype_dirty) return 0;
    PoolLayout L;
    L.narr = ctx->narr;
    for (int a = 0; a < ctx->narr; a++) {
        L.off[a] = ctx->arr[a].off;
        L.n[a] = ctx->arr[a].n;
        L.n_real[a] = ctx->arr[a].n_real;
    }
    if (ctx->pool_end > 0) {
        k_fill_ptype<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(ctx->ptype,
                                                                                  ctx->pool_end, L);
        LAUNCH_CHECK();
    }
    ctx->ptype_dirty = false;
    return 0;
}

// the main stream waits for what the peer protocol left running on the communication stream
static int sync_comm(b200sph_ctx *ctx)
{
    if (!ctx->comm_pending) return 0;
    ctx->comm_pending = false;
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_red, 0));
    return 0;
}

static int materialise_pending(b200sph_ctx *ctx);
// every entry point starts here; all but those of the time step's fast path (pair_pass, eos,
// nnps_update, the WCSPH stages, update_domain, the dt reductions: keep_init) first run a
// deferred initialize or half step, and, as they may write accelerations, no longer count on
// the spare acceleration set matching the slots
static int ensure_pool(b200sph_ctx *ctx, bool join = true, bool keep_init = false)
{
    if (join) {
        int rc0 = sync_comm(ctx);
        if (rc0) return rc0;
    }
    if (!keep_init) {
        if (int rci = materialise_pending(ctx)) return rci;
        ctx->acc_differ = ~0u;
    }
    if (ctx->pool_cap == 0) {
        int64_t caps[B200SPH_MAX_ARRAYS];
        for (int a = 0; a < ctx->narr; a++) caps[a] = std::max(ctx->arr[a].cap, ctx->arr[a].n);
        int rc = pool_layout(ctx, caps);
        if (rc) return rc;
    }
    return refresh_ptype(ctx);
}

static int device_scan(b200sph_ctx *ctx, const uint32_t *in, uint32_t *out, int64_t n)
{
    const int64_t nb = cdiv(n, SCAN_TILE);
    if (int rc = grow(ctx, ctx->blk_sums, nb, nb + 1024)) return rc;
    k_scan_tiles<<<(unsigned)nb, SCAN_THREADS, 0, ctx->stream>>>(in, out, n, ctx->blk_sums);
    LAUNCH_CHECK();
    if (nb > 1) {
        k_scan_sums<<<1, SCAN_THREADS, 0, ctx->stream>>>(ctx->blk_sums, nb);
        LAUNCH_CHECK();
        k_scan_add<<<(unsigned)nb, SCAN_THREADS, 0, ctx->stream>>>(out, n, ctx->blk_sums);
        LAUNCH_CHECK();
    }
    return 0;
}

// Per-phase device timing without host syncs: event pairs are recorded on the
// context's stream and only resolved (cudaEventElapsedTime) in get_stats.
struct PhaseTimer {
    b200sph_ctx *ctx;
    int slot;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    PhaseTimer(b200sph_ctx *c, int s) : ctx(c) { start(s); }
    ~PhaseTimer() { stop(); }
    void to(int s) { stop(); start(s); }   // ends this phase; what follows is timed into slot s
    void start(int s);
    void stop();
};


void PhaseTimer::start(int s)
{
    slot = s;
    if (!ctx->profiling || (ctx->profiling == 2 && slot != 1)) return;
    for (cudaEvent_t *e : {&e0, &e1}) {
        if (!ctx->ev_pool.empty()) {
            *e = ctx->ev_pool.back();
            ctx->ev_pool.pop_back();
        } else {
            cudaEventCreate(e);
        }
    }
    cudaEventRecord(e0, ctx->stream);
}
void PhaseTimer::stop()
{
    if (!e0) return;
    cudaEventRecord(e1, ctx->stream);
    ctx->pending.push_back({e0, e1, slot});
    e0 = e1 = nullptr;
}

// The (kernel, dim) pairs the templated pair-walking kernels are instantiated for: every kernel
// in 1-3 dimensions except WendlandQuintic in 1-D (b200sph_set_kernel refuses it).  `launch`
// gets them as std::integral_constant<int, K> and std::integral_constant<int, DIM>.
template <class F> static int with_kernel_dim(b200sph_ctx *ctx, int kernel, int dim, const char *who, F &&launch)
{
    using std::integral_constant;
    switch (kernel * 4 + dim) {
#define KD(K, D) \
    case K * 4 + D: return launch(integral_constant<int, K>(), integral_constant<int, D>());
        KD(0, 1) KD(0, 2) KD(0, 3) KD(1, 2) KD(1, 3) KD(2, 1) KD(2, 2) KD(2, 3) KD(3, 1) KD(3, 2) KD(3, 3)
#undef KD
    default: return set_err(ctx, "%s: unsupported kernel/dim combination", who);
    }
}
template <class F> static int with_kernel_dim(b200sph_ctx *ctx, const char *who, F &&launch)
{
    return with_kernel_dim(ctx, ctx->kernel, ctx->dim, who, launch);
}

// with the elastic-dynamics arrays allocated the deviatoric stress travels too: a ghost is a
// source of group 2 (and, with SolidProgram.ghost_group1, a destination of group 1), and a
// migrating particle takes s and its stage copy s0 along
static inline int halo_nf(const b200sph_ctx *ctx) { return elastic_allocated(ctx) ? B200SPH_HALO_FIELDS_SOLID : B200SPH_HALO_FIELDS; }
static inline int migrate_nf(const b200sph_ctx *ctx) { return elastic_allocated(ctx) ? B200SPH_MIGRATE_FIELDS_SOLID : B200SPH_MIGRATE_FIELDS; }

// the halo kernels are instantiated for either field count; `launch` gets it as
// std::integral_constant<int, NF>
template <class F> static int with_halo_fields(const b200sph_ctx *ctx, F &&launch)
{
    if (halo_nf(ctx) == B200SPH_HALO_FIELDS) return launch(std::integral_constant<int, B200SPH_HALO_FIELDS>());
    return launch(std::integral_constant<int, B200SPH_HALO_FIELDS_SOLID>());
}

// the fields StageArgs, StageTvfArgs and StageSolidArgs have in common, by name (devdt: the
// kernel takes dt from the time-control block)
template <class S> static void stage_args(b200sph_ctx *ctx, S &sa, int arr, int which, double dt, bool devdt)
{
    sa.x = f64_ptr(ctx, B200SPH_X); sa.y = f64_ptr(ctx, B200SPH_Y); sa.z = f64_ptr(ctx, B200SPH_Z);
    sa.u = f64_ptr(ctx, B200SPH_U); sa.v = f64_ptr(ctx, B200SPH_V); sa.w = f64_ptr(ctx, B200SPH_W);
    sa.x0 = f64_ptr(ctx, B200SPH_X0); sa.y0 = f64_ptr(ctx, B200SPH_Y0); sa.z0 = f64_ptr(ctx, B200SPH_Z0);
    sa.u0 = f64_ptr(ctx, B200SPH_U0); sa.v0 = f64_ptr(ctx, B200SPH_V0); sa.w0 = f64_ptr(ctx, B200SPH_W0);
    sa.au = f32_ptr(ctx, B200SPH_AU); sa.av = f32_ptr(ctx, B200SPH_AV); sa.aw = f32_ptr(ctx, B200SPH_AW);
    sa.ax = f32_ptr(ctx, B200SPH_AX); sa.ay = f32_ptr(ctx, B200SPH_AY); sa.az = f32_ptr(ctx, B200SPH_AZ);
    sa.ptype = ctx->ptype;
    sa.pool_end = ctx->pool_end;
    sa.arr = arr;
    sa.which = which;
    sa.f = which == 1 ? 0.5 * dt : dt;
    sa.tc = devdt ? ctx->tc : nullptr;
}

// ---- the deferred initialize ----------------------------------------------------------------
// WCSPHStep.initialize of every array (WCSPHTVDRK3Step's is the same) copies x .. rho into
// x0 .. rho0.  When the stage that follows will be the fused kernel, stage_impl only records it
// (init_pending) and that kernel takes it as it goes (do_init): one sweep over the state less per
// step.  Stage 1 of a context without ghosts does not even copy: the host exchanges the two sets
// of buffers in ctx->prop (init_by_rename), so that the state the initialize saw goes by
// x0 .. rho0 where it lies and the kernel writes the stepped state into the buffers that now go
// by x .. rho (INIT_RENAMED); 56 B per particle less to write.  Otherwise the kernel copies
// (INIT_COPY).  The one rule: whatever could observe the copy not being made yet -- reads x0 .. rho0,
// writes x .. rho, applies EOS calls to the pool's rho (eos_flush, pack_state), changes the
// particle set or the stream -- runs it here first, as k_stage(0) on the state as it is, which is
// the state the initialize saw.  ensure_pool does so for every entry point outside the fast path.
// Only the fused stage 1 renames; every other way to the initialize copies.
static int init_materialise(b200sph_ctx *ctx)
{
    if (!ctx->init_pending) return 0;
    ctx->init_pending = false;
    StageArgs sa;
    stage_args(ctx, sa, -1, 0, 0.0, false);
    sa.rho = f64_ptr(ctx, B200SPH_RHO); sa.rho0 = f64_ptr(ctx, B200SPH_RHO0); sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    if (ctx->pool_end > 0) {
        k_stage<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    return 0;
}

// ---- the deferred half step ------------------------------------------------------------------
// WCSPHStep.stage2 computes q = q0 + dt aq from x0 .. rho0 and the second evaluation's
// accelerations, and that evaluation reads the predicted state from the 32-byte records: in a
// step that nothing observes between the stages nobody reads the predicted x .. w, nor the p / cs
// that stage 1 formed from rho0 (stage 2 writes them again); the predicted rho only feeds stage
// 2's EOS calls, and stage 2 can form it again as stage 1 did.  So the fused stage 1 that takes
// the initialize by renaming (init_by_rename) and writes the 32-byte records leaves them unwritten
// (half_pending, 64 B per particle less to store) and the host keeps what forms them: the stage's
// factor and its EOS calls.  The pair pass of the second evaluation writes its accelerations into
// the spare set (acc_swap), so that the first evaluation's stay readable.  The one rule: whatever
// could observe x .. rho or p / cs not being written yet -- reads or changes them, a full build, a
// push, a change of the particle set, the stream or the time-control block, any stage but the
// fused stage 2 -- runs half_materialise first; the fused stage 2 clears half_pending without it.
static int half_materialise(b200sph_ctx *ctx)
{
    if (!ctx->half_pending) return 0;
    ctx->half_pending = false;
    StageArgs sa;
    stage_args(ctx, sa, -1, 1, 0.0, false);
    sa.f = ctx->half_f;
    sa.tc = ctx->half_tc;
    sa.rho = f64_ptr(ctx, B200SPH_RHO); sa.rho0 = f64_ptr(ctx, B200SPH_RHO0); sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    if (ctx->acc_swapped) {
        sa.arho = ctx->acc_spare[0];
        sa.au = ctx->acc_spare[1]; sa.av = ctx->acc_spare[2]; sa.aw = ctx->acc_spare[3];
        sa.ax = ctx->acc_spare[4]; sa.ay = ctx->acc_spare[5]; sa.az = ctx->acc_spare[6];
        ctx->acc_swapped = false;
    }
    if (ctx->pool_end > 0) {
        k_half_materialise<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(
            sa, f32_ptr(ctx, B200SPH_P), f32_ptr(ctx, B200SPH_CS), ctx->half_eos, ctx->half_EP);
        LAUNCH_CHECK();
    }
    ctx->n_half_materialised++;
    return 0;
}

// a deferred half step, then a deferred initialize (the two are never pending together)
static int materialise_pending(b200sph_ctx *ctx)
{
    if (int rc = half_materialise(ctx)) return rc;
    return init_materialise(ctx);
}

// The accelerations a pair pass writes, as ACC_* bits: au .. aw of array d (bit d), ax .. az
// (bit 8 + d) and arho (bit 16 + d).  k_pair_list_r32 writes them exactly where the Group has a
// momentum / an XSPH / a continuity equation for the destination's array; for the other pair
// kernels the mask takes every array.
enum { ACC_UVW = 0, ACC_XYZ = 8, ACC_RHO = 16 };
static unsigned acc_writes(const b200sph_ctx *ctx, const b200sph_pair_program *prog, bool r32)
{
    if (!r32) return ~0u;
    unsigned w = 0;
    for (int d = 0; d < ctx->narr; d++) {
        unsigned bits = 0;
        for (int s = 0; s < ctx->narr; s++) bits |= prog->eqmask[d][s];
        if (bits & B200SPH_EQ_MOMENTUM) w |= 1u << (ACC_UVW + d);
        if (bits & B200SPH_EQ_XSPH) w |= 1u << (ACC_XYZ + d);
        if (bits & B200SPH_EQ_CONTINUITY) w |= 1u << (ACC_RHO + d);
    }
    return w;
}

// The pair pass of the second evaluation (writes: acc_writes) while a half step is pending gets
// the spare arho, au .. az: the two sets exchange names, as x / x0 do in init_by_rename, and the set of
// the first evaluation stays in acc_spare for half_materialise.  A particle whose accelerations
// this pass does not write must find the same values under the new names: where the sets may
// differ there, the slots are copied into the spare set first (once, while the same passes run).
static int acc_swap(b200sph_ctx *ctx, unsigned writes)
{
    const size_t n = (size_t)ctx->pool_cap;
    for (Buf<float> &b : ctx->acc_spare)
        if (int rc = grow(ctx, b, n, n)) return rc;
    if (ctx->acc_differ & ~writes) {
        for (int k = 0; k < 7; k++)
            CU(cudaMemcpyAsync(ctx->acc_spare[k], ctx->prop[B200SPH_ARHO + k], sizeof(float) * (size_t)ctx->pool_end,
                               cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->acc_differ = 0;
    }
    for (int k = 0; k < 7; k++) {
        void *slot = ctx->prop[B200SPH_ARHO + k];
        ctx->prop[B200SPH_ARHO + k] = ctx->acc_spare[k].p;
        ctx->acc_spare[k].p = (float *)slot;
    }
    ctx->acc_swapped = true;
    return 0;
}

// the pair counter of a pass that reports its pair count (pairs_out != null)
static int pairs_arm(b200sph_ctx *ctx, const int64_t *pairs_out, unsigned long long **counter)
{
    if (!pairs_out) return 0;
    CU(cudaMemsetAsync(ctx->counter, 0, 8, ctx->stream));
    *counter = ctx->counter;
    return 0;
}
static int pairs_read(b200sph_ctx *ctx, int64_t *pairs_out)
{
    if (!pairs_out) return 0;
    CU(cudaMemcpyAsync(ctx->counter_host, ctx->counter, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    *pairs_out = (int64_t)ctx->counter_host[0];
    ctx->stats.pairs += *pairs_out;
    return 0;
}

static double kernel_fac(int kernel, int dim)
{
    const double pi = 3.14159265358979323846;
    switch (kernel) {
    case 0: return dim == 3 ? 1.0 / pi : (dim == 2 ? 10.0 / (7.0 * pi) : 2.0 / 3.0);  // kernels.py:57-65
    case 1: return dim == 2 ? 7.0 / (4.0 * pi) : 21.0 / (16.0 * pi);                  // kernels.py:291-299
    case 2: return dim == 1 ? 1.0 / 120.0 : (dim == 2 ? 7.0 / (478.0 * pi) : 1.0 / (120.0 * pi));  // kernels.py:1071-1079
    default: return std::pow(1.0 / std::sqrt(pi), dim);                                // kernels.py:852-858
    }
}
static double kernel_radius_scale(int kernel)
{
    return (kernel == B200SPH_KERNEL_QUINTIC_SPLINE || kernel == B200SPH_KERNEL_GAUSSIAN) ? 3.0 : 2.0;
}
static double kernel_deltap(int kernel)
{
    switch (kernel) {
    case 0: return 2. / 3;
    case 1: return 0.5;
    case 2: return 0.759298480738450;
    default: return 0.70710678118654746;
    }
}

extern "C" {

static int eos_flush(b200sph_ctx *ctx, cudaStream_t on_comm_stream = nullptr);
static void free_peer_pending(b200sph_ctx *ctx);
static void generic_unload_all(b200sph_ctx *ctx);

int b200sph_abi_version(void) { return B200SPH_ABI_VERSION; }

int b200sph_create(int device, b200sph_ctx **out)
{
    if (!out) return -1;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev) {
        fprintf(stderr, "b200sph_create: no usable CUDA device %d (found %d) -- this library has "
                        "no CPU fallback\n", device, ndev);
        return -2;
    }
    b200sph_ctx *ctx = new b200sph_ctx();
    ctx->device = device;
    memset(&ctx->grid, 0, sizeof(ctx->grid));
    memset(&ctx->eos_pending, 0, sizeof(ctx->eos_pending));
    memset(&ctx->eos_last, 0, sizeof(ctx->eos_last));
    memset(&ctx->stats, 0, sizeof(ctx->stats));
    *out = ctx;
    CU(cudaSetDevice(device));
    CU(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    ctx->own_stream = true;
    if (const char *e = getenv("B200SPH_PAIR_KERNEL")) {
        if (!strcmp(e, "warp")) ctx->force_kernel = 1;
        else if (strcmp(e, "list") && e[0]) {
            fprintf(stderr, "b200sph: B200SPH_PAIR_KERNEL must be list or warp\n");
            delete ctx;
            *out = nullptr;
            return -3;
        }
    }
    if (const char *e = getenv("B200SPH_FUSE")) ctx->fuse = atoi(e) != 0;
    if (const char *e = getenv("B200SPH_ZORDER")) ctx->zorder = atoi(e) != 0;
    if (const char *e = getenv("B200SPH_PROACTIVE")) ctx->proactive = atoi(e) != 0;
    if (const char *e = getenv("B200SPH_SKIN")) ctx->skin = ctx->skin_max = std::max(0.0, atof(e));
    if (const char *e = getenv("B200SPH_SKIN_ADAPT")) ctx->skin_adapt = atoi(e) != 0;
    if (const char *e = getenv("B200SPH_RECORDS")) ctx->rec48_forced = atoi(e) == 48;
    ctx->skin_min = std::min(ctx->skin_min, ctx->skin_max);
    int rc;
    if ((rc = grow(ctx, ctx->red_u32, 4, 4)) || (rc = grow(ctx, ctx->red_u32_host, 4, 4)) ||
        (rc = grow(ctx, ctx->drift_host, 4, 4)) || (rc = grow(ctx, ctx->red, 16, 16)) ||
        (rc = grow(ctx, ctx->red_host, 16, 16)) || (rc = grow(ctx, ctx->counter, 8, 8)) ||
        (rc = grow(ctx, ctx->counter_host, 8, 8)))
        return rc;
    CU(cudaEventCreateWithFlags(&ctx->drift_evt, cudaEventDisableTiming));
    return 0;
}

// the buffers free themselves (Buf) when ctx is deleted, after the streams have drained
int b200sph_destroy(b200sph_ctx *ctx)
{
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (void *b : ctx->prop) cudaFree(b);
    generic_unload_all(ctx);
    for (int i = 0; i < 2; i++)
        if (ctx->tc_evt[i]) cudaEventDestroy(ctx->tc_evt[i]);
    if (ctx->drift_evt) cudaEventDestroy(ctx->drift_evt);
    for (auto &pe : ctx->pending) { cudaEventDestroy(pe.e0); cudaEventDestroy(pe.e1); }
    for (auto e : ctx->ev_pool) cudaEventDestroy(e);
    if (ctx->snap_stream) { cudaStreamSynchronize(ctx->snap_stream); cudaStreamDestroy(ctx->snap_stream); }
    if (ctx->snap_ready) cudaEventDestroy(ctx->snap_ready);
    if (ctx->snap_done) cudaEventDestroy(ctx->snap_done);
    for (int r = 0; r < ctx->peer_world; r++)
        if (r != ctx->peer_rank && ctx->peer_boxes[r]) cudaIpcCloseMemHandle(ctx->peer_boxes[r]);
    if (ctx->comm_stream) { cudaStreamSynchronize(ctx->comm_stream); cudaStreamDestroy(ctx->comm_stream); }
    if (ctx->red_stream) { cudaStreamSynchronize(ctx->red_stream); cudaStreamDestroy(ctx->red_stream); }
    if (ctx->ev_pushed) cudaEventDestroy(ctx->ev_pushed);
    if (ctx->ev_red) cudaEventDestroy(ctx->ev_red);
    free_peer_pending(ctx);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return 0;
}

const char *b200sph_last_error(b200sph_ctx *ctx)
{
    if (!ctx) return "null context";
    std::lock_guard<std::mutex> lk(ctx->err_mu);
    ctx->err_out = ctx->err;     // a stable copy: another thread may be writing the next message
    return ctx->err_out.c_str();
}

int b200sph_set_stream(b200sph_ctx *ctx, void *s)
{
    CU(cudaSetDevice(ctx->device));
    if (int rci = materialise_pending(ctx)) return rci;
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->own_stream) CU(cudaStreamDestroy(ctx->stream));
    if (s) {
        ctx->stream = (cudaStream_t)s;
        ctx->own_stream = false;
    } else {
        CU(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        ctx->own_stream = true;
    }
    return 0;
}

int b200sph_synchronize(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    if (int rcj = sync_comm(ctx)) return rcj;
    CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int b200sph_add_array(b200sph_ctx *ctx, const char *name, int64_t n, int64_t n_real, int64_t capacity)
{
    if (ctx->narr >= B200SPH_MAX_ARRAYS) return set_err(ctx, "too many particle arrays (max %d)", B200SPH_MAX_ARRAYS);
    if (n < 0 || n_real < 0 || n_real > n) return set_err(ctx, "add_array: bad sizes n=%lld n_real=%lld", (long long)n, (long long)n_real);
    CU(cudaSetDevice(ctx->device));
    if (int rci = materialise_pending(ctx)) return rci;   // (before the layout moves)
    const int a = ctx->narr;
    ctx->arr[a].name = name ? name : "";
    ctx->arr[a].n = n;
    ctx->arr[a].n_real = n_real;
    ctx->arr[a].cap = std::max<int64_t>(capacity, n);
    ctx->arr[a].off = 0;
    ctx->narr++;
    if (ctx->pool_cap > 0) {  // pool already built: re-layout, preserving data of older arrays
        int64_t caps[B200SPH_MAX_ARRAYS];
        const int64_t n_new = ctx->arr[a].n;
        ctx->arr[a].n = 0;  // nothing to move for the new array
        for (int k = 0; k < ctx->narr; k++) caps[k] = ctx->arr[k].cap;
        int rc = pool_layout(ctx, caps);
        ctx->arr[a].n = n_new;
        if (rc) return rc;
    }
    set_changed(ctx);
    return a;
}

int b200sph_resize_array(b200sph_ctx *ctx, int arr, int64_t n, int64_t n_real)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "resize_array: bad array %d", arr);
    if (n < 0 || n_real < 0 || n_real > n) return set_err(ctx, "resize_array: bad sizes");
    CU(cudaSetDevice(ctx->device));
    if (int rci = materialise_pending(ctx)) return rci;
    { int rc0 = eos_flush(ctx); if (rc0) return rc0; }
    if (ctx->pool_cap == 0) {
        ctx->arr[arr].cap = std::max(ctx->arr[arr].cap, n);
    } else {
        int rc = ensure_capacity(ctx, arr, n);
        if (rc) return rc;
    }
    ctx->arr[arr].n = n;
    ctx->arr[arr].n_real = n_real;
    set_changed(ctx);
    return 0;
}

int b200sph_get_array_size(b200sph_ctx *ctx, int arr, int64_t *n, int64_t *n_real)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "get_array_size: bad array %d", arr);
    if (n) *n = ctx->arr[arr].n;
    if (n_real) *n_real = ctx->arr[arr].n_real;
    return 0;
}

static int check_range(b200sph_ctx *ctx, int arr, int64_t start, int64_t count)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "bad array index %d", arr);
    if (start < 0 || count < 0 || start + count > ctx->arr[arr].n)
        return set_err(ctx, "range [%lld, %lld) outside array '%s' of %lld particles", (long long)start,
                       (long long)(start + count), ctx->arr[arr].name.c_str(), (long long)ctx->arr[arr].n);
    return 0;
}

static int ensure_stage(b200sph_ctx *ctx, int64_t count) { return grow(ctx, ctx->stage_buf, count, count + 1024); }

// a named elastic-dynamics or user property: allocated (zeroed) the first time anything names it,
// the elastic-dynamics properties as one group with their stress records
static int ensure_prop(b200sph_ctx *ctx, int prop)
{
    const PropGroup g = prop_kind(prop).group;
    if (g == GROUP_POOL || ctx->prop[prop]) return 0;
    const size_t alloc = (size_t)std::max<int64_t>(ctx->pool_cap, 32);
    for (int p = 0; p < N_PROP_SLOTS; p++) {
        if (p != prop && (g == GROUP_USER || prop_kind(p).group != g)) continue;
        const size_t esz = prop_kind(p).size();
        CU(cudaMalloc(&ctx->prop[p], esz * alloc));
        CU(cudaMemsetAsync(ctx->prop[p], 0, esz * alloc, ctx->stream));
    }
    if (g == GROUP_ELASTIC)
        for (Buf<float4> *r : {&ctx->T01, &ctx->T2R, &ctx->R2})
            if (int rc = grow(ctx, *r, alloc, alloc)) return rc;
    return 0;
}

int b200sph_push_f64(b200sph_ctx *ctx, int arr, int prop, const double *host, int64_t start, int64_t count)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = check_range(ctx, arr, start, count))) return rc;
    // naming an elastic-dynamics property allocates that pool even for an empty array: every
    // rank of a slab decomposition must agree on the message layout (b200sph_halo_layout)
    if ((rc = ensure_prop(ctx, prop))) return rc;
    if (count == 0) return 0;
    const int64_t o = ctx->arr[arr].off + start;
    const PropType t = prop_kind(prop).type;
    if (t == PROP_F64) {
        CU(cudaMemcpyAsync(f64_ptr(ctx, prop) + o, host, 8 * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
    } else if (t == PROP_F32) {
        if ((rc = ensure_stage(ctx, count))) return rc;
        CU(cudaMemcpyAsync(ctx->stage_buf, host, 8 * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
        k_f64_to_f32<<<(unsigned)cdiv(count, 256), 256, 0, ctx->stream>>>(ctx->stage_buf, f32_ptr(ctx, prop) + o, count);
        LAUNCH_CHECK();
    } else {
        return set_err(ctx, "push_f64: property id %d is not a floating point property", prop);
    }
    // the host buffer is borrowed only for this call
    if (!ctx->async_copies) CU(cudaStreamSynchronize(ctx->stream));
    // new positions / smoothing lengths for the SAME particles: the next nnps_update
    // measures the drift against the current neighbour build and reuses it if it can
    if (prop == B200SPH_H) h_changed(ctx);
    else if (prop <= B200SPH_Z) positions_changed(ctx);
    else if (prop == B200SPH_M) m_changed(ctx);
    state_changed(ctx);
    return 0;
}

static int require_confirmed(b200sph_ctx *ctx, const char *who);
int b200sph_pull_f64(b200sph_ctx *ctx, int arr, int prop, double *host, int64_t start, int64_t count)
{
    if (int rcc = require_confirmed(ctx, "pull_f64")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if ((rc = check_range(ctx, arr, start, count))) return rc;
    if (count == 0) return 0;
    const int64_t o = ctx->arr[arr].off + start;
    if ((rc = ensure_prop(ctx, prop))) return rc;
    const PropType t = prop_kind(prop).type;
    if (t == PROP_F64) {
        CU(cudaMemcpyAsync(host, f64_ptr(ctx, prop) + o, 8 * (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
    } else if (t == PROP_F32) {
        if ((rc = ensure_stage(ctx, count))) return rc;
        k_f32_to_f64<<<(unsigned)cdiv(count, 256), 256, 0, ctx->stream>>>(f32_ptr(ctx, prop) + o, ctx->stage_buf, count);
        LAUNCH_CHECK();
        CU(cudaMemcpyAsync(host, ctx->stage_buf, 8 * (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
        return set_err(ctx, "pull_f64: property id %d is not a floating point property", prop);
    }
    if (!ctx->async_copies) CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int b200sph_push_u32(b200sph_ctx *ctx, int arr, int prop, const uint32_t *host, int64_t start, int64_t count)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = check_range(ctx, arr, start, count))) return rc;
    if (prop_kind(prop).type != PROP_U32) return set_err(ctx, "push_u32: property id %d is not an integer property", prop);
    if (count == 0) return 0;
    CU(cudaMemcpyAsync(u32_ptr(ctx, prop) + ctx->arr[arr].off + start, host, 4 * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
    if (!ctx->async_copies) CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int b200sph_pull_u32(b200sph_ctx *ctx, int arr, int prop, uint32_t *host, int64_t start, int64_t count)
{
    if (int rcc = require_confirmed(ctx, "pull_u32")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = check_range(ctx, arr, start, count))) return rc;
    if (prop_kind(prop).type != PROP_U32) return set_err(ctx, "pull_u32: property id %d is not an integer property", prop);
    if (count == 0) return 0;
    CU(cudaMemcpyAsync(host, u32_ptr(ctx, prop) + ctx->arr[arr].off + start, 4 * (size_t)count, cudaMemcpyDeviceToHost, ctx->stream));
    if (!ctx->async_copies) CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int b200sph_device_ptr(b200sph_ctx *ctx, int arr, int prop, void **out)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "device_ptr: bad array %d", arr);
    if ((rc = ensure_prop(ctx, prop))) return rc;
    const PropKind pk = prop_kind(prop);
    if (pk.type == PROP_NONE) return set_err(ctx, "device_ptr: bad property %d", prop);
    *out = (char *)ctx->prop[prop] + pk.size() * (size_t)ctx->arr[arr].off;
    return 0;
}

// ---- asynchronous output snapshot ---------------------------------------------------
// take: device-to-device copies (fp32 properties widened) into a private buffer, in stream
// order -- the time loop goes on at once; fetch: device-to-host on a second stream, from
// any host thread; release: lets the next take overwrite the buffer.
int b200sph_snapshot_take(b200sph_ctx *ctx, int nseg, const int *arr, const int *prop, const int64_t *count)
{
    if (int rcc = require_confirmed(ctx, "snapshot_take")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (ctx->snap_open) return set_err(ctx, "snapshot_take: the previous snapshot was not released");
    if (nseg < 1) return set_err(ctx, "snapshot_take: no segments");
    if (!ctx->snap_stream) {
        CU(cudaStreamCreateWithFlags(&ctx->snap_stream, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&ctx->snap_ready, cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&ctx->snap_done, cudaEventDisableTiming));
    } else {
        // the copies of the previous snapshot must have left the buffer
        CU(cudaStreamWaitEvent(ctx->stream, ctx->snap_done, 0));
    }
    int64_t total = 0;
    for (int i = 0; i < nseg; i++) {
        if (arr[i] == -1) {  // the time-control block {dt, t, ...}
            if (!ctx->tc) return set_err(ctx, "snapshot_take: no time-control block");
            if (count[i] < 1 || count[i] > 8) return set_err(ctx, "snapshot_take: the time-control block has 8 doubles");
        } else if ((rc = check_range(ctx, arr[i], 0, count[i]))) return rc;
        total += std::max<int64_t>(count[i], 1);
    }
    if ((rc = grow(ctx, ctx->snap_buf, total, total + total / 8 + 1024))) return rc;
    ctx->snap_off.assign(nseg, 0), ctx->snap_len.assign(nseg, 0), ctx->snap_u32.assign(nseg, 0);
    int64_t at = 0;
    for (int i = 0; i < nseg; i++) {
        const int64_t n = count[i];
        ctx->snap_off[i] = at, ctx->snap_len[i] = n;
        double *dst = ctx->snap_buf + at;
        at += std::max<int64_t>(n, 1);
        if (n == 0) continue;
        if (arr[i] == -1) {
            CU(cudaMemcpyAsync(dst, ctx->tc, 8 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
            continue;
        }
        const int64_t o = ctx->arr[arr[i]].off;
        const int pr = prop[i];
        if ((rc = ensure_prop(ctx, pr))) return rc;
        const PropType t = prop_kind(pr).type;
        if (t == PROP_F64) {
            CU(cudaMemcpyAsync(dst, f64_ptr(ctx, pr) + o, 8 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
        } else if (t == PROP_F32) {
            k_f32_to_f64<<<(unsigned)cdiv(n, 256), 256, 0, ctx->stream>>>(f32_ptr(ctx, pr) + o, dst, n);
            LAUNCH_CHECK();
        } else if (t == PROP_U32) {
            ctx->snap_u32[i] = 1;
            CU(cudaMemcpyAsync(dst, u32_ptr(ctx, pr) + o, 4 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
        } else {
            return set_err(ctx, "snapshot_take: bad property %d", pr);
        }
    }
    CU(cudaEventRecord(ctx->snap_ready, ctx->stream));
    ctx->snap_open = true;
    return 0;
}

int b200sph_snapshot_fetch(b200sph_ctx *ctx, int seg, void *host, int64_t count)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->snap_open) return set_err(ctx, "snapshot_fetch: no snapshot");
    if (seg < 0 || seg >= (int)ctx->snap_len.size() || count != ctx->snap_len[seg])
        return set_err(ctx, "snapshot_fetch: segment %d does not hold %lld elements", seg, (long long)count);
    if (count == 0) return 0;
    CU(cudaStreamWaitEvent(ctx->snap_stream, ctx->snap_ready, 0));
    CU(cudaMemcpyAsync(host, ctx->snap_buf + ctx->snap_off[seg], (ctx->snap_u32[seg] ? 4 : 8) * (size_t)count,
                       cudaMemcpyDeviceToHost, ctx->snap_stream));
    CU(cudaStreamSynchronize(ctx->snap_stream));
    return 0;
}

int b200sph_snapshot_release(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->snap_open) return 0;
    CU(cudaEventRecord(ctx->snap_done, ctx->snap_stream));
    ctx->snap_open = false;
    return 0;
}

int b200sph_set_kernel(b200sph_ctx *ctx, int kernel, int dim)
{
    if (kernel < 0 || kernel > 3) return set_err(ctx, "set_kernel: unknown kernel id %d", kernel);
    if (dim < 1 || dim > 3) return set_err(ctx, "set_kernel: dim must be 1, 2 or 3");
    if (kernel == B200SPH_KERNEL_WENDLAND_QUINTIC && dim == 1)
        return set_err(ctx, "WendlandQuintic: Dim 1 not supported");  // kernels.py:289-290
    ctx->kernel = kernel;
    ctx->dim = dim;
    ctx->radius_scale = kernel_radius_scale(kernel);
    h_changed(ctx);   // (the cell size is radius_scale hmax)
    build_invalid(ctx);
    return 0;
}

static int run_minmax(b200sph_ctx *ctx, int do_xyz, int do_h)
{
    k_red_init<<<1, 32, 0, ctx->stream>>>(ctx->red);
    LAUNCH_CHECK();
    ctx->red_armed = true;   // (slots 9, 11, 12 are not touched by k_reduce_minmax)
    ctx->dt_reduced = false;
    if (ctx->pool_end > 0) {
        const unsigned nb = (unsigned)std::min<int64_t>(cdiv(ctx->pool_end, 256), REDUCE_BLOCKS);
        k_reduce_minmax<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z),
                                                     f64_ptr(ctx, B200SPH_H), ctx->ptype, ctx->pool_end, do_xyz, do_h, ctx->red);
        LAUNCH_CHECK();
    }
    CU(cudaMemcpyAsync(ctx->red_host, ctx->red, 16 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// h and m of every particle uniform?  k_reduce_minmax over (h, m, m) into slots 0..5 only:
// the dt factors a fused stage2 may have reduced into slots 9, 11, 12 stay where they are
static int hm_uniformity(b200sph_ctx *ctx)
{
    if (ctx->hm_known) return 0;
    static const long long init[6] = {d2o(1e300), d2o(-1e300), d2o(1e300), d2o(-1e300), d2o(1e300), d2o(-1e300)};
    CU(cudaMemcpyAsync(ctx->red, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    if (ctx->pool_end > 0) {
        const unsigned nb = (unsigned)std::min<int64_t>(cdiv(ctx->pool_end, 256), REDUCE_BLOCKS);
        k_reduce_minmax<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_H), f64_ptr(ctx, B200SPH_M), f64_ptr(ctx, B200SPH_M),
                                                     nullptr, ctx->ptype, ctx->pool_end, 1, 0, ctx->red);
        LAUNCH_CHECK();
    }
    CU(cudaMemcpyAsync(ctx->red_host, ctx->red, 4 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const double h0 = o2d(ctx->red_host[0]), h1 = o2d(ctx->red_host[1]);
    const double m0 = o2d(ctx->red_host[2]), m1 = o2d(ctx->red_host[3]);
    ctx->h_uniform = (h0 == h1 && h0 > 0.0) ? h0 : NAN;
    ctx->m_uniform = (m0 == m1) ? m0 : NAN;
    ctx->hm_known = true;
    return 0;
}

int b200sph_set_domain(b200sph_ctx *ctx, const double lo[3], const double hi[3], const int periodic[3])
{
    if ((periodic[0] || periodic[1] || periodic[2]) && (ctx->mirror[0] || ctx->mirror[1] || ctx->mirror[2]))
        return set_err(ctx, "set_domain: mirror planes in a periodic domain are not supported");
    for (int d = 0; d < 3; d++) {
        if (periodic[d] && !(hi[d] > lo[d])) return set_err(ctx, "Invalid domain limits!");  // nnps_base.pyx:352-355
        ctx->periodic[d] = periodic[d] != 0;
        ctx->dom_lo[d] = lo[d];
        ctx->dom_hi[d] = hi[d];
    }
    build_invalid(ctx);
    return 0;
}

static inline bool mirror_any(const b200sph_ctx *ctx) { return ctx->mirror[0] || ctx->mirror[1] || ctx->mirror[2]; }
static int mirror_create(b200sph_ctx *ctx);
static int mirror_refresh(b200sph_ctx *ctx);

int b200sph_set_mirror(b200sph_ctx *ctx, const int mirror[3], double n_layers)
{
    if (!(n_layers >= 1.0)) return set_err(ctx, "set_mirror: n_layers must be >= 1 (the images must cover one kernel support)");
    for (int d = 0; d < 3; d++) {
        if (mirror[d] && !(ctx->dom_hi[d] > ctx->dom_lo[d])) return set_err(ctx, "Invalid domain limits!");
    }
    // the reference mirrors the periodic ghosts it has just created as well (nnps_base.pyx:471-480);
    // here periodic images are never materialised, so the combination is refused
    if ((mirror[0] || mirror[1] || mirror[2]) && (ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2]))
        return set_err(ctx, "set_mirror: mirror planes in a periodic domain are not supported");
    for (int d = 0; d < 3; d++) ctx->mirror[d] = mirror[d] != 0;
    ctx->mirror_layers = n_layers;
    ctx->mirror_built = false;
    build_invalid(ctx);
    return 0;
}

int b200sph_update_domain(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    // (only the periodic wrap reads the state; the rest is h)
    int rc = ensure_pool(ctx, true, !(ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2]));
    if (rc) return rc;
    if (ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2]) {
        // _box_wrap_periodic, nnps_base.pyx:699-743 (part of DomainManager.update)
        if ((rc = eos_flush(ctx))) return rc;
        GridDev D;
        for (int d = 0; d < 3; d++) {
            D.xmin[d] = ctx->dom_lo[d];
            D.cell[d] = ctx->dom_hi[d] - ctx->dom_lo[d];
            D.nc[d] = 1;
            D.periodic[d] = ctx->periodic[d];
        }
        D.zorder = 0;
        if (ctx->pool_end > 0) {
            k_box_wrap<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z),
                                                                                   ctx->ptype, ctx->pool_end, D);
            LAUNCH_CHECK();
        }
        particles_moved(ctx);
    }
    if (ctx->domain_valid && !ctx->h_dirty) return 0;  // h untouched since the last reduction
    PhaseTimer pt(ctx, 2);
    if ((rc = run_minmax(ctx, 0, 1))) return rc;
    // nnps_base.pyx:942-978
    double hmin = o2d(ctx->red_host[6]), hmax = o2d(ctx->red_host[7]);
    int64_t ntot = 0;
    for (int a = 0; a < ctx->narr; a++) ntot += ctx->arr[a].n;
    if (ntot == 0) { hmax = -1.0; hmin = 1.7976931348623157e308; }
    double cell = ctx->radius_scale * hmax;
    ctx->hmin_scaled = ctx->radius_scale * hmin;
    if (cell < 1e-6) cell = 1.0;
    if (cell != ctx->cell_size) positions_changed(ctx);
    ctx->cell_size = cell;
    ctx->domain_valid = true;
    ctx->h_dirty = false;
    return 0;
}

// 2 |dx|max + k dh: the part of the skin the drift since the build has used up, in length
// units, from a host copy of the fp32 max-reduction red_u32[0..1] (|dx|^2 and dh as bits)
static double drift_need(const b200sph_ctx *ctx, const unsigned *raw)
{
    float d2, dh;
    memcpy(&d2, &raw[0], 4);
    memcpy(&dh, &raw[1], 4);
    return 2.0 * std::sqrt((double)d2) + ctx->radius_scale * (double)dh;
}

// 2 |dx|max + k dh <= S, with a 2 % safety margin for the fp32 measurement
static bool drift_within_skin(b200sph_ctx *ctx, const unsigned *raw) { return drift_need(ctx, raw) <= 0.98 * ctx->S_abs; }

// Skin controller, part 2 (part 1 adapts the skin geometrically from the lifetime of the build
// that has just ended, see nnps_update).  A build is RETIRED -- rebuilt although it is valid --
//  * when it has lived 3 L* evaluations with more than the minimum skin (a quiet flow must
//    converge to the minimum skin), or
//  * early, after SKIN_PROBE evaluations, when the drift measured so far says the skin is far too
//    generous: with d = drift per evaluation, a skin s lives L(s) = 0.98 s cell / d evaluations,
//    and L(s) = L*(s) = kappa / s gives s* = sqrt(kappa d / (0.98 cell)).  s* < 0.7 s: rebuild
//    now with s* (a rebuild costs ~3 evaluations' worth of the list entries it removes per
//    evaluation; the first build of a run is always made blind, with the maximum skin).
#define SKIN_PROBE 6
static bool retire_build(b200sph_ctx *ctx)
{
    if (!ctx->skin_adapt || !(ctx->skin > ctx->skin_min)) return false;
    if (ctx->evals_since_build >= 3.0 * SKIN_KAPPA / ctx->skin) return true;
    if (ctx->evals_since_build == SKIN_PROBE && ctx->drift_hist[1] >= 0.0 && ctx->cell_size > 0.0) {
        const double d = ctx->drift_hist[1] * ctx->S_abs / (double)SKIN_PROBE;
        const double s_opt = std::min(ctx->skin_max, std::max(ctx->skin_min, std::sqrt(SKIN_KAPPA * d / (0.98 * ctx->cell_size))));
        if (s_opt < 0.7 * ctx->skin) {
            ctx->skin_next = s_opt;
            return true;
        }
    }
    return false;
}

// k_pack_pos_light: the packed positions refreshed in the frozen order of the build, their drift
// since the build max-reduced into red_u32[0..1] after the first `clear` words of red_u32 are
// zeroed (0: the drift is added to what red_u32 holds)
static int pack_positions_light(b200sph_ctx *ctx, int clear)
{
    if (int rc = half_materialise(ctx)) return rc;
    if (clear) CU(cudaMemsetAsync(ctx->red_u32, 0, clear * sizeof(unsigned), ctx->stream));
    k_pack_pos_light<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(
        f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z), f64_ptr(ctx, B200SPH_H), ctx->perm, ctx->skey,
        ctx->n_sorted, ctx->G, ctx->A0, ctx->A, ctx->AB, ctx->red_u32);
    ctx->ab_stale = false;   // (k_pack_pos_light writes the position half of AB)
    LAUNCH_CHECK();
    return 0;
}

// light path of nnps_update: same sorted order, same cell frames, fresh positions;
// returns 1 if the persistent lists are still valid, 0 if a full rebuild is needed
static int nnps_light_update(b200sph_ctx *ctx)
{
    if (ctx->n_sorted <= 0) return 1;
    if (ctx->drift_ok) {
        // the drift was just measured by b200sph_nnps_drift or peer_begin (multi-GPU: the
        // decision to keep the build is collective); only refresh the packed positions, no host sync
        ctx->drift_ok = false;
        drift_consumed(ctx);
        if (ctx->packed_valid) return 1;   // peer_begin packed them, peer_recv kept the ghosts current
        if (int rc = pack_positions_light(ctx, 0)) return rc;
        return 1;
    }
    if (!(ctx->packed_valid && ctx->drift_measured)) {   // (the fused stage kernel packs and measures)
        if (int rc = pack_positions_light(ctx, 4)) return rc;
    }
    drift_consumed(ctx);
    ctx->packed_valid = true;
    if (ctx->defer_check) {
        // optimistic: carry on as if the lists were valid; b200sph_nnps_confirm reads the
        // measurement after the evaluation has been enqueued (no idle GPU while we wait)
        CU(cudaMemcpyAsync(ctx->drift_host, ctx->red_u32, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaEventRecord(ctx->drift_evt, ctx->stream));
        ctx->check_pending = true;
        return 1;
    }
    CU(cudaMemcpyAsync(ctx->red_u32_host, ctx->red_u32, 4 * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return drift_within_skin(ctx, ctx->red_u32_host) ? 1 : 0;
}

static int confirm_pending(b200sph_ctx *ctx, int *redo)
{
    *redo = 0;
    if (!ctx->check_pending) return 0;
    CU(cudaSetDevice(ctx->device));
    CU(cudaEventSynchronize(ctx->drift_evt));
    ctx->check_pending = false;
    ctx->drift_hist[0] = ctx->drift_hist[1];
    ctx->drift_hist[1] = ctx->S_abs > 0.0 ? drift_need(ctx, ctx->drift_host) / ctx->S_abs : 2.0;
    if (!drift_within_skin(ctx, ctx->drift_host)) {
        // the evaluation that followed used stale lists: force the full rebuild
        build_invalid(ctx);
        ctx->n_light_updates--;
        ctx->n_deferred_failed++;
        *redo = 1;
        ctx->iisph_restore = ctx->iisph_spec;
        ctx->gtvf_restore = ctx->gtvf_spec;
    }
    ctx->iisph_spec = false;
    ctx->gtvf_spec = false;
    return 0;
}
// entry points that consume the results of an evaluation must not run on an
// unconfirmed deferred update
static int require_confirmed(b200sph_ctx *ctx, const char *who)
{
    if (!ctx->check_pending) return 0;
    int redo = 0, rc = confirm_pending(ctx, &redo);
    if (rc) return rc;
    if (redo)
        return set_err(ctx, "%s: the deferred drift check of the last nnps_update failed and was never confirmed "
                            "(call b200sph_nnps_confirm after the evaluation and repeat it when asked to)", who);
    return 0;
}

int b200sph_nnps_confirm(b200sph_ctx *ctx, int *redo) { return confirm_pending(ctx, redo); }

int b200sph_nnps_update_deferred(b200sph_ctx *ctx)
{
    ctx->defer_check = true;
    const int rc = b200sph_nnps_update(ctx);
    ctx->defer_check = false;
    return rc;
}

int b200sph_nnps_update(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    // with the peer protocol's refresh in flight the only thing this call may do without
    // waiting for it is to accept the build the ranks have (speculatively) agreed to keep
    int rc = ensure_pool(ctx, !(ctx->comm_pending && ctx->drift_ok && ctx->packed_valid && reusable_build(ctx) &&
                                !ctx->eos_any && ctx->domain_valid && !ctx->check_pending),
                     true);
    if (rc) return rc;
    if (ctx->check_pending) {   // update after update without an evaluation in between
        int redo = 0;
        if ((rc = confirm_pending(ctx, &redo))) return rc;
    }
    if ((rc = eos_flush(ctx))) return rc;
    if (!ctx->domain_valid && (rc = b200sph_update_domain(ctx))) return rc;
    PhaseTimer pt(ctx, 0);

    int64_t ntot0 = 0;
    for (int a = 0; a < ctx->narr; a++) ntot0 += ctx->arr[a].n;
    const bool use_lists = lists_usable(ctx, ntot0);
    // deferred check + a build whose drift, extrapolated by its last increment, would exceed
    // the skin at THIS evaluation: rebuild now rather than after an evaluation on stale lists
    bool expiring = false;
    if (ctx->proactive && ctx->defer_check && !ctx->drift_ok && ctx->drift_hist[1] >= 0.0) {
        const double r1 = ctx->drift_hist[1], r0 = ctx->drift_hist[0];
        const double step = r0 >= 0.0 ? std::max(r1 - r0, 0.0) : r1;
        expiring = r1 + step > 0.98;
        if (expiring && use_lists && reusable_build(ctx)) ctx->n_proactive++;
    }
    if (use_lists && reusable_build(ctx) && !expiring &&
        !(!ctx->drift_ok && retire_build(ctx))) {
        // mirror images: the same ghosts, current values (the set is re-selected with the lists)
        if (mirror_any(ctx) && ctx->mirror_built && (rc = mirror_refresh(ctx))) return rc;
        rc = nnps_light_update(ctx);
        if (rc < 0) return rc;
        if (rc == 1) {
            ctx->n_light_updates++;
            ctx->evals_since_build++;
            ctx->grid_valid = true;   // (state_packed is left alone: whatever changed the state cleared it)
            return 0;
        }
    }
    // skin controller (see SKIN_KAPPA): a build that outlived 1.5 L* was built with too
    // generous a skin, one that lasted less than L* / 1.5 with too small a one; builds that
    // reach 3 L* are retired so that a quiet flow converges to the minimum skin
    if (use_lists && ctx->skin_adapt && ctx->lists_valid && ctx->evals_since_build > 0) {
        const double lstar = SKIN_KAPPA / ctx->skin;
        if (ctx->skin_next > 0.0) ctx->skin = ctx->skin_next;     // measured (retire_build)
        else if (ctx->evals_since_build >= 1.5 * lstar) ctx->skin = std::max(ctx->skin_min, ctx->skin * 0.75);
        else if (ctx->evals_since_build < lstar / 1.5) ctx->skin = std::min(ctx->skin_max, ctx->skin * 1.33);
    }
    if ((rc = half_materialise(ctx))) return rc;   // the full build reads x, y, z
    ctx->skin_next = -1.0;
    ctx->evals_since_build = 0;
    lists_stale(ctx);
    ctx->drift_ok = false;
    ctx->drift_hist[0] = ctx->drift_hist[1] = -1.0;
    ctx->n_full_builds++;
    if (mirror_any(ctx)) {
        // _create_ghosts_mirror (nnps_base.pyx:506-689) -- here once per list build, not per update
        if ((rc = mirror_create(ctx))) return rc;
        if (!ctx->domain_valid && (rc = b200sph_update_domain(ctx))) return rc;
    }

    int64_t ntot = 0;
    for (int a = 0; a < ctx->narr; a++) ntot += ctx->arr[a].n;
    if (ntot >= (1LL << 32) - 1) return set_err(ctx, "more than 2^32-2 particles: indices are 32-bit (as in the reference)");

    // _compute_bounds nnps_base.pyx:1520-1575
    if ((rc = run_minmax(ctx, 1, 0))) return rc;
    double mn[3], mx[3], l[3];
    for (int d = 0; d < 3; d++) {
        mn[d] = ntot ? o2d(ctx->red_host[2 * d]) : 1e100;
        mx[d] = ntot ? o2d(ctx->red_host[2 * d + 1]) : -1e100;
        l[d] = mx[d] - mn[d];
    }
    for (int d = 0; d < 3; d++) {
        mn[d] -= l[d] * 0.01;
        mx[d] += l[d] * 0.01;
    }
    const double domain_size = std::max(std::max(l[0], l[1]), l[2]);
    if (ctx->last_domain_size > 1e-16 && domain_size > 2.0 * ctx->last_domain_size)
        fprintf(stderr, "b200sph WARNING: Domain size has increased by a large amount. "
                        "Particles are probably diverging, please check your code!\n");
    ctx->last_domain_size = domain_size;
    if (std::fabs(mx[0] - mn[0]) < 1e-12 && std::fabs(mx[1] - mn[1]) < 1e-12 && std::fabs(mx[2] - mn[2]) < 1e-12)
        for (int d = 0; d < 3; d++) {
            mn[d] -= 0.5;
            mx[d] += 0.5;
        }
    // the reference's grid: _get_number_of_cells / _count_occupied_cells
    // linked_list_nnps.pyx:293-343 (reported by get_grid; the 2^28 guard is honoured)
    int nc_ref[3];
    {
        const double cs1 = 1. / ctx->cell_size;
        for (int d = 0; d < 3; d++) {
            const double v = std::ceil(cs1 * (mx[d] - mn[d]));
            if (!(v < 2147483647.0)) return set_err(ctx, "ERROR: LinkedListNNPS requires too many cells along axis %d", d);
            nc_ref[d] = (int)v;
            if (nc_ref[d] < 0) return set_err(ctx, "LinkedListNNPS: Number of cells is negative");
            if (nc_ref[d] == 0) nc_ref[d] = 1;
        }
        const double ncells_d = (double)nc_ref[0] * (double)nc_ref[1] * (double)nc_ref[2];
        if (ncells_d > (double)(1LL << 28))
            return set_err(ctx, "ERROR: LinkedListNNPS requires too many cells (%.0f).", ncells_d);
    }
    b200sph_grid_info &gi = ctx->grid;
    gi.cell_size = ctx->cell_size;
    gi.hmin = ctx->hmin_scaled;
    for (int d = 0; d < 3; d++) {
        gi.xmin[d] = mn[d];
        gi.xmax[d] = mx[d];
        gi.ncells[d] = nc_ref[d];
    }
    gi.n_cells = (int64_t)nc_ref[0] * nc_ref[1] * nc_ref[2];
    gi.n_particles = ntot;

    // the internal grid: cells widened by the skin when the persistent lists are used
    ctx->S_abs = use_lists ? ctx->skin * ctx->cell_size : 0.0;
    ctx->cell_int = ctx->cell_size + ctx->S_abs;
    int nc[3];
    double cellv[3];
    for (int d = 0; d < 3; d++) {
        if (ctx->periodic[d]) {
            // a periodic axis is tiled EXACTLY by cells not smaller than the cut-off, so
            // that the image shift of a wrapped neighbour cell is a whole number of cells
            const double L = ctx->dom_hi[d] - ctx->dom_lo[d];
            if (!(L >= ctx->cell_int))
                return set_err(ctx, "periodic axis %d: the domain (%g) is smaller than the interaction range + skin (%g)", d, L, ctx->cell_int);
            mn[d] = ctx->dom_lo[d];
            mx[d] = ctx->dom_hi[d];
            nc[d] = std::max(1, (int)std::floor(L / ctx->cell_int));
            cellv[d] = L / nc[d];
        } else {
            nc[d] = (int)std::ceil((mx[d] - mn[d]) / ctx->cell_int);
            if (nc[d] <= 0) nc[d] = 1;
            cellv[d] = ctx->cell_int;
        }
    }
    int64_t ncells = (int64_t)nc[0] * nc[1] * nc[2];
    if (ncells > (1LL << 28)) return set_err(ctx, "ERROR: LinkedListNNPS requires too many cells (%lld).", (long long)ncells);
    // Z-curve over the cell rows: the row table is padded to a power of two per axis (the
    // unused rows are empty cells); a grid whose padding would be excessive stays row-major
    int zorder = 0;
    if (ctx->zorder) {
        int bits = 0;
        while ((1 << bits) < std::max(nc[1], nc[2])) bits++;
        const int64_t padded = ((int64_t)1 << (2 * bits)) * nc[0];
        if (bits <= 15 && padded <= (1LL << 27) && padded <= 8 * ncells + (1 << 20)) {
            zorder = 1;
            ncells = padded;
        }
    }

    for (Buf<uint32_t> *b : {&ctx->cell_cnt, &ctx->cell_start})
        if ((rc = grow(ctx, *b, ncells + 2, ncells + ncells / 2 + 1024))) return rc;
    GridDev &G = ctx->G;
    for (int d = 0; d < 3; d++) {
        G.xmin[d] = mn[d];
        G.nc[d] = nc[d];
    }
    for (int d = 0; d < 3; d++) {
        G.cell[d] = cellv[d];
        G.periodic[d] = ctx->periodic[d] ? 1 : 0;
    }
    G.zorder = zorder;

    CU(cudaMemsetAsync(ctx->cell_cnt, 0, 4 * (size_t)(ncells + 1), ctx->stream));
    ctx->n_sorted = ntot;
    if (ctx->pool_end > 0) {
        const unsigned nb = (unsigned)cdiv(ctx->pool_end, 256);
        k_cell_count<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z),
                                                  ctx->ptype, ctx->pool_end, G, ctx->key_of, ctx->off_in, ctx->cell_cnt);
        LAUNCH_CHECK();
    }
    if ((rc = device_scan(ctx, ctx->cell_cnt, ctx->cell_start, ncells + 1))) return rc;
    if (ctx->pool_end > 0 && ntot > 0) {
        const unsigned nb = (unsigned)cdiv(ctx->pool_end, 256);
        k_scatter<<<nb, 256, 0, ctx->stream>>>(ctx->key_of, ctx->off_in, ctx->ptype, ctx->pool_end, ctx->cell_start, ctx->perm_tmp);
        LAUNCH_CHECK();
        const unsigned ns = (unsigned)cdiv(ntot, 256);
        k_canon<<<ns, 256, 0, ctx->stream>>>(ctx->perm_tmp, ctx->key_of, ctx->cell_start, ntot, ctx->perm, ctx->skey, ctx->rank);
        LAUNCH_CHECK();
        k_pack_pos<<<ns, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z), f64_ptr(ctx, B200SPH_H),
                                                ctx->perm, ctx->skey, ntot, G, ctx->A, ctx->AB, ctx->ptype, ctx->stype);
        LAUNCH_CHECK();
        if (use_lists)
            CU(cudaMemcpyAsync(ctx->A0, ctx->A, 16 * (size_t)ntot, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    ctx->topo_dirty = false;
    ctx->grid_valid = true;
    ctx->ab_stale = false;   // (k_pack_pos wrote AB)
    state_changed(ctx);   // new sorted slots
    return 0;
}

// With ghosts in the build (slab decomposition) the CTAs of the list consumers are split
// into the ones that do not depend on a ghost -- they may run while the halo of the
// evaluation is still in flight -- and the rest (k_chunk_classify).  Called by build_lists,
// which has marked the chunks stale.
static int split_chunks(b200sph_ctx *ctx)
{
    int64_t nghost = 0;
    for (int a = 0; a < ctx->narr; a++) nghost += ctx->arr[a].n - ctx->arr[a].n_real;
    const int64_t n = ctx->n_sorted, nchunks = cdiv(n, LIST_NT);
    if (nghost == 0 || n <= 0 || (size_t)nchunks + 1 > ctx->flag_a.cap) return 0;
    const int64_t reserve = nchunks + nchunks / 4 + 64;
    int rc;
    for (Buf<uint32_t> *b : {&ctx->chunk_boundary, &ctx->chunk_interior})
        if ((rc = grow(ctx, *b, nchunks, reserve))) return rc;
    if ((rc = grow(ctx, ctx->sflag, nchunks * LIST_NT, reserve * LIST_NT))) return rc;
    if ((rc = refresh_ptype(ctx))) return rc;
    k_sorted_ghost_flag<<<(unsigned)cdiv(n, 256), 256, 0, ctx->stream>>>(ctx->ptype, ctx->perm, n, ctx->sflag);
    LAUNCH_CHECK();
    k_chunk_classify<<<(unsigned)nchunks, LIST_NT, 0, ctx->stream>>>(ctx->cnt, ctx->lst, ctx->capg, ctx->sflag, n, ctx->flag_a);
    LAUNCH_CHECK();
    if ((rc = device_scan(ctx, ctx->flag_a, ctx->flag_b, nchunks + 1))) return rc;
    uint32_t nb = 0;
    CU(cudaMemcpyAsync(&nb, ctx->flag_b + nchunks, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    k_chunk_split<<<(unsigned)cdiv(nchunks, 256), 256, 0, ctx->stream>>>(nchunks, ctx->flag_a, ctx->flag_b, ctx->chunk_boundary, ctx->chunk_interior);
    LAUNCH_CHECK();
    ctx->n_chunk_boundary = nb;
    ctx->n_chunk_interior = nchunks - nb;
    ctx->chunks_valid = true;
    return 0;
}

// (re)build the persistent neighbour lists for the current build.  want[d] (8 bits per source
// type; null: everything) = the (destination, source) type pairs the caller has equations for:
// the lists are filtered with the union of what has been asked for since the particle set last
// changed, so that e.g. a wall particle's wall neighbours -- for which the WCSPH Group has no
// equation -- are never stored, gathered or tested (they were a quarter of the list entries of
// a wall-heavy slab).
static bool lists_cover(const b200sph_ctx *ctx, const unsigned long long *want)
{
    for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) {
        const unsigned long long w = want ? want[d] : ~0ull;
        for (int sx = 0; sx < B200SPH_MAX_ARRAYS; sx++)
            if (((w >> (8 * sx)) & 0xFFull) && !((ctx->list_mask[d] >> (8 * sx)) & 0xFFull)) return false;
    }
    return true;
}
static int build_lists(b200sph_ctx *ctx, const unsigned long long *want)
{
    lists_stale(ctx);
    for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) {
        const unsigned long long w = want ? want[d] : ~0ull;
        for (int sx = 0; sx < B200SPH_MAX_ARRAYS; sx++)
            if ((w >> (8 * sx)) & 0xFFull) ctx->list_mask[d] |= 0xFFull << (8 * sx);
    }
    const int64_t n = ctx->n_sorted;
    ListBuildArgs la;
    la.A = ctx->A; la.cell_start = ctx->cell_start; la.skey = ctx->skey;
    la.n = n;
    la.ncx = ctx->G.nc[0]; la.ncy = ctx->G.nc[1]; la.ncz = ctx->G.nc[2];
    la.cellx = (float)ctx->G.cell[0]; la.celly = (float)ctx->G.cell[1]; la.cellz = (float)ctx->G.cell[2];
    la.zorder = ctx->G.zorder;
    la.px = ctx->G.periodic[0]; la.py = ctx->G.periodic[1]; la.pz = ctx->G.periodic[2];
    const bool per = la.px || la.py || la.pz;
    la.kr = (float)ctx->radius_scale;
    la.S = (float)ctx->S_abs;
    la.cnt = ctx->cnt;
    la.max_count = ctx->red_u32 + 2;
    for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) la.emask[d] = ctx->list_mask[d];
    la.stype = ctx->stype;
    const unsigned nb = (unsigned)cdiv(n, LB_WARPS * 32);
    const int64_t nblk = cdiv(n, 32);
    for (int attempt = 0; attempt < 4; attempt++) {
        const bool count_only = ctx->capg == 0;
        if (!count_only) {
            const int64_t need = nblk * ctx->capg * 32;
            if (int rc = grow(ctx, ctx->lst, need, need + need / 8)) return rc;
        }
        la.lst = count_only ? nullptr : ctx->lst.p;
        la.capg = ctx->capg;
        CU(cudaMemsetAsync(ctx->red_u32 + 2, 0, sizeof(unsigned), ctx->stream));
        if (per) k_list_build<true><<<nb, LB_WARPS * 32, 0, ctx->stream>>>(la);
        else k_list_build<false><<<nb, LB_WARPS * 32, 0, ctx->stream>>>(la);
        LAUNCH_CHECK();
        CU(cudaMemcpyAsync(ctx->red_u32_host + 2, ctx->red_u32 + 2, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        const int maxc = (int)ctx->red_u32_host[2];
        if (!count_only && maxc <= ctx->capg) {
            ctx->lists_valid = true;
            ctx->n_list_builds++;
            return split_chunks(ctx);
        }
        // (re)size: a little head-room so that later rebuilds usually fit in one pass
        ctx->capg = ((int)(maxc * 1.15) + 8 + 7) / 8 * 8;
    }
    return set_err(ctx, "neighbour list build did not converge");
}

// The neighbour lists a pass walks, filtered for `want` (see build_lists).  Refused with the
// caller's message when the lists cannot index the particles; rebuilt, as neighbour-search
// time, when the current ones do not cover `want`.
static int prepare_lists(b200sph_ctx *ctx, const unsigned long long *want, const char *refusal)
{
    if (!lists_usable(ctx, ctx->n_sorted)) return set_err(ctx, "%s", refusal);
    if (ctx->lists_valid && lists_cover(ctx, want)) return 0;
    PhaseTimer pt(ctx, 0);
    return build_lists(ctx, want);
}

int b200sph_get_grid(b200sph_ctx *ctx, b200sph_grid_info *out)
{
    if (!ctx->grid_valid) return set_err(ctx, "get_grid: the NNPS has not been updated");
    *out = ctx->grid;
    return 0;
}

// the pool side of the EOS calls a pair pass left for the fused stage kernel, stand-alone
static int eos_pool_flush(b200sph_ctx *ctx, cudaStream_t s)
{
    if (!ctx->eos_pool_any) return 0;
    if (ctx->pool_end > 0) {
        k_eos_tab<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, s>>>(f64_ptr(ctx, B200SPH_RHO), f32_ptr(ctx, B200SPH_P),
                                                                      f32_ptr(ctx, B200SPH_CS), ctx->ptype, ctx->pool_end, ctx->eos_pool);
        LAUNCH_CHECK();
    }
    ctx->eos_pool_any = false;
    return 0;
}

// run the pending equation-of-state calls stand-alone (something needs rho/p/cs now, or the
// packed records already hold them: the pool side of a speculated EOS) -- one launch
static int eos_flush(b200sph_ctx *ctx, cudaStream_t on_comm_stream)
{
    if (!ctx->eos_any && !ctx->eos_pool_any) return 0;
    // ghost rho may be in the middle of a refresh: wait for it -- unless the caller puts
    // this launch on the communication stream itself, behind the scatter
    if (!on_comm_stream)
        if (int rcj = sync_comm(ctx)) return rcj;
    if (int rci = materialise_pending(ctx)) return rci;   // (it copies the rho of before these calls)
    cudaStream_t s = on_comm_stream ? on_comm_stream : ctx->stream;
    if (int rcp = eos_pool_flush(ctx, s)) return rcp;   // (the older calls first)
    if (!ctx->eos_any) return 0;
    EosTab &E = ctx->eos_pending;
    if (ctx->pool_end > 0) {
        k_eos_tab<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, s>>>(
            f64_ptr(ctx, B200SPH_RHO), f32_ptr(ctx, B200SPH_P), f32_ptr(ctx, B200SPH_CS), ctx->ptype, ctx->pool_end, E);
        LAUNCH_CHECK();
    }
    memset(E.on, 0, sizeof(E.on));
    ctx->eos_any = false;
    return 0;
}

// Every reader of the position half of AB other than k_pair_list_r32 calls this first: after
// k_stage_pack wrote the 32-byte records, the positions are in R only.
static int ab_positions(b200sph_ctx *ctx)
{
    if (!ctx->ab_stale) return 0;
    if (ctx->n_sorted > 0) {
        k_rec32_positions<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(ctx->R, f64_ptr(ctx, B200SPH_H), ctx->perm,
                                                                                       ctx->n_sorted, ctx->AB);
        LAUNCH_CHECK();
    }
    ctx->ab_stale = false;
    return 0;
}

static int pack_state(b200sph_ctx *ctx)
{
    if (int rc = ab_positions(ctx)) return rc;   // (k_pack_rec32 reads them)
    if (int rc = half_materialise(ctx)) return rc;   // (the packers read u, v, w, p, cs)
    // the packers read the pool's rho and apply eos_pending to it (eos_flush's order: the
    // initialize, then the older calls)
    if (ctx->eos_any || ctx->eos_pool_any) {
        if (int rc = init_materialise(ctx)) return rc;
        if (int rc = eos_pool_flush(ctx, ctx->stream)) return rc;
    }
    if (ctx->rec32 && ctx->n_sorted > 0) {
        // (every particle is sorted: no ghosts, so the pool side of the EOS calls is complete)
        k_pack_rec32<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(
            f64_ptr(ctx, B200SPH_U), f64_ptr(ctx, B200SPH_V), f64_ptr(ctx, B200SPH_W), f64_ptr(ctx, B200SPH_RHO), f32_ptr(ctx, B200SPH_P),
            f32_ptr(ctx, B200SPH_CS), ctx->ptype, ctx->perm, ctx->n_sorted, ctx->AB, ctx->R, ctx->eos_pending, ctx->rec32_eos);
        LAUNCH_CHECK();
        memset(ctx->eos_pending.on, 0, sizeof(ctx->eos_pending.on));
        ctx->eos_any = false;
    } else if (ctx->n_sorted > 0) {
        k_pack_state<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(
            f64_ptr(ctx, B200SPH_U), f64_ptr(ctx, B200SPH_V), f64_ptr(ctx, B200SPH_W), f64_ptr(ctx, B200SPH_M), f64_ptr(ctx, B200SPH_RHO),
            f32_ptr(ctx, B200SPH_P), f32_ptr(ctx, B200SPH_CS), ctx->ptype, ctx->perm, ctx->n_sorted, ctx->B, ctx->C, ctx->AB,
            ctx->eos_pending, ctx->eos_any ? 1 : 0);
        LAUNCH_CHECK();
        memset(ctx->eos_pending.on, 0, sizeof(ctx->eos_pending.on));
        ctx->eos_any = false;
    }
    ctx->state_packed = true;
    ctx->spec_records = false;
    return 0;
}

int64_t b200sph_get_neighbors(b200sph_ctx *ctx, int dst_arr, int src_arr, int64_t d_idx, uint32_t *out, int64_t cap)
{
    if (int rcc = require_confirmed(ctx, "get_neighbors")) return rcc;
    CU(cudaSetDevice(ctx->device));
    if (!ctx->grid_valid) return set_err(ctx, "get_neighbors: call nnps_update first");
    if (dst_arr < 0 || dst_arr >= ctx->narr || src_arr < 0 || src_arr >= ctx->narr) return set_err(ctx, "get_neighbors: bad array index");
    if (d_idx < 0 || d_idx >= ctx->arr[dst_arr].n) return set_err(ctx, "get_neighbors: d_idx out of range");
    int rc;
    if (ctx->rec32) ctx->rec32 = false, state_changed(ctx);   // k_neighbors reads the 48-byte records
    if ((rc = ab_positions(ctx))) return rc;
    if (!ctx->state_packed && (rc = pack_state(ctx))) return rc;
    uint32_t s32 = 0;
    CU(cudaMemcpyAsync(&s32, ctx->rank + ctx->arr[dst_arr].off + d_idx, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const int64_t dcap = std::max<int64_t>(cap, 1);
    Buf<uint32_t> dout;
    if ((rc = grow(ctx, dout, dcap, dcap))) return rc;
    k_neighbors<<<1, 32, 0, ctx->stream>>>(ctx->AB, ctx->C, ctx->cell_start, ctx->skey, ctx->perm, (long long)s32, src_arr,
                                           (long long)ctx->arr[src_arr].off, ctx->G, (float)(ctx->radius_scale * ctx->radius_scale),
                                           dout, cap, ctx->counter + 1);
    LAUNCH_CHECK();
    CU(cudaMemcpyAsync(ctx->counter_host + 1, ctx->counter + 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const int64_t n = (int64_t)ctx->counter_host[1];
    const int64_t ncopy = std::min(n, cap);
    if (ncopy > 0) {
        CU(cudaMemcpy(out, dout, 4 * (size_t)ncopy, cudaMemcpyDeviceToHost));
        std::sort(out, out + ncopy);
    }
    return n;
}

static int arr_range(b200sph_ctx *ctx, int arr, int real_only, int64_t *lo, int64_t *hi)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "bad array index %d", arr);
    *lo = ctx->arr[arr].off;
    *hi = ctx->arr[arr].off + (real_only ? ctx->arr[arr].n_real : ctx->arr[arr].n);
    return 0;
}

int b200sph_eos(b200sph_ctx *ctx, int arr, int hg, double rho0, double c0, double gamma, double p0, int real_only)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, false, true);   // only book-keeping here: a halo in flight stays in flight
    if (rc) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "bad array index %d", arr);
    EosTab &E = ctx->eos_pending;
    // a second call for the same array before the first was applied, or a build that
    // is not valid (no sorted order to pack): run what is pending now
    if ((E.on[arr] || !ctx->grid_valid) && (rc = eos_flush(ctx))) return rc;
    E.on[arr] = 1; E.hg[arr] = hg; E.real_only[arr] = real_only;
    E.rho0[arr] = rho0; E.c0[arr] = c0; E.gamma[arr] = gamma; E.p0[arr] = p0;
    ctx->eos_any = true;
    if (!ctx->grid_valid && (rc = eos_flush(ctx))) return rc;
    // the fused stage kernel may have applied exactly this call to the packed records
    // already (it repeats the last evaluation's calls); pair_pass checks that ALL of them
    // were confirmed before it trusts the records
    const EosTab &L = ctx->eos_last;
    if (ctx->spec_records && ctx->state_packed && ctx->eos_last_valid && L.on[arr] && L.hg[arr] == hg &&
        L.real_only[arr] == real_only && L.rho0[arr] == rho0 && L.c0[arr] == c0 && L.gamma[arr] == gamma && L.p0[arr] == p0) {
        ctx->spec_confirmed |= 1u << arr;
    } else {
        state_changed(ctx);
        ctx->spec_records = false;
    }
    return 0;
}

int b200sph_ferrari_h(b200sph_ctx *ctx, int arr, double hdx, int dim, int real_only)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    int64_t lo, hi;
    if ((rc = arr_range(ctx, arr, real_only, &lo, &hi))) return rc;
    PhaseTimer pt(ctx, 2);
    if (hi > lo) {
        k_ferrari<<<(unsigned)cdiv(hi - lo, 256), 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_H), f64_ptr(ctx, B200SPH_M), f64_ptr(ctx, B200SPH_RHO), lo, hi, hdx, 1.0 / dim);
        LAUNCH_CHECK();
    }
    h_changed(ctx);
    return 0;
}

// ---- generic-equation fallback (pysph_b200/codegen.py; SURVEY.md 8f-4) ---------------------
// Kernels generated from user Equation bodies and compiled by NVRTC are loaded through the
// driver API, which is looked up at first use (the library itself links the runtime only, so
// that it loads -- and fails loudly at the first CUDA call -- on a box without a driver).
#include <dlfcn.h>
#ifndef B200SPH_HOST_EMULATION
struct DriverApi {
    void *lib = nullptr;
    int (*ModuleLoadData)(void **, const void *) = nullptr;
    int (*ModuleGetFunction)(void **, void *, const char *) = nullptr;
    int (*ModuleUnload)(void *) = nullptr;
    int (*LaunchKernel)(void *, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void *, void **, void **) = nullptr;
    int (*GetErrorString)(int, const char **) = nullptr;
};
static DriverApi g_drv;
static int driver_api(b200sph_ctx *ctx)
{
    if (g_drv.lib) return 0;
    void *lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return set_err(ctx, "generic equations: cannot load libcuda.so.1 (%s)", dlerror());
    DriverApi d;
    d.ModuleLoadData = (int (*)(void **, const void *))dlsym(lib, "cuModuleLoadData");
    d.ModuleGetFunction = (int (*)(void **, void *, const char *))dlsym(lib, "cuModuleGetFunction");
    d.ModuleUnload = (int (*)(void *))dlsym(lib, "cuModuleUnload");
    d.LaunchKernel = (int (*)(void *, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void *, void **, void **))dlsym(lib, "cuLaunchKernel");
    d.GetErrorString = (int (*)(int, const char **))dlsym(lib, "cuGetErrorString");
    if (!d.ModuleLoadData || !d.ModuleGetFunction || !d.ModuleUnload || !d.LaunchKernel)
        return set_err(ctx, "generic equations: libcuda.so.1 lacks the module API");
    d.lib = lib;
    g_drv = d;
    return 0;
}
static const char *drv_err(int e)
{
    const char *m = nullptr;
    if (g_drv.GetErrorString) g_drv.GetErrorString(e, &m);
    return m ? m : "unknown driver error";
}
#endif

static void generic_unload_all(b200sph_ctx *ctx)
{
    for (void *m : ctx->gen_modules) {
        if (!m) continue;
#ifdef B200SPH_HOST_EMULATION
        dlclose(m);
#else
        if (g_drv.ModuleUnload) g_drv.ModuleUnload(m);
#endif
    }
    ctx->gen_modules.clear();
}

int b200sph_user_property(b200sph_ctx *ctx, int prop)
{
    CU(cudaSetDevice(ctx->device));
    if (prop_kind(prop).group != GROUP_USER) return set_err(ctx, "user_property: ids %d..%d", B200SPH_USER0, B200SPH_USER0 + B200SPH_MAX_USER - 1);
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    return ensure_prop(ctx, prop);
}

int b200sph_generic_load(b200sph_ctx *ctx, const void *image, int64_t size)
{
    CU(cudaSetDevice(ctx->device));
    if (!image || size <= 0) return set_err(ctx, "generic_load: empty image");
    void *mod = nullptr;
#ifdef B200SPH_HOST_EMULATION
    // the emulated library runs kernels that a TEST compiled for the host: the "image" is the
    // path of that shared object
    mod = dlopen((const char *)image, RTLD_NOW | RTLD_LOCAL);
    if (!mod) return set_err(ctx, "generic_load: %s", dlerror());
#else
    int rc = driver_api(ctx);
    if (rc) return rc;
    CU(cudaFree(0));   // the runtime's primary context is current on this thread from here on
    const int e = g_drv.ModuleLoadData(&mod, image);
    if (e) return set_err(ctx, "generic_load: cuModuleLoadData: %s", drv_err(e));
#endif
    ctx->gen_modules.push_back(mod);
    return (int)ctx->gen_modules.size() - 1;
}

// One phase (0 initialize, 1 loop, 2 post_loop) of one destination array of a generated Group
// kernel.  src_mask: the source arrays of its loop bodies; writes: bit 0 a body stores to
// x / y / z / h, bit 1 to any other property the packed records are made from.
int b200sph_generic_launch(b200sph_ctx *ctx, int module, const char *kernel, int dest_arr, int phase, unsigned src_mask,
                           int real_only, double t, double dt, int writes)
{
    if (int rcc = require_confirmed(ctx, "generic_launch")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (module < 0 || module >= (int)ctx->gen_modules.size()) return set_err(ctx, "generic_launch: bad module handle %d", module);
    if (dest_arr < 0 || dest_arr >= ctx->narr || phase < 0 || phase > 2) return set_err(ctx, "generic_launch: bad destination / phase");
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "generic equations run on one GPU (no slab decomposition)");
    if (!ctx->grid_valid) return set_err(ctx, "generic_launch: the NNPS is stale (particles were pushed/resized); call nnps_update first");
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    const bool ranged = ctx->dst_ranged;   // one-shot, as for pair_pass: every launch names its own
    ctx->dst_ranged = false;
    static const char no_lists[] = "generic equations need the neighbour-list path";
    if (ctx->n_sorted > 0 && !lists_usable(ctx, ctx->n_sorted)) return set_err(ctx, "%s", no_lists);
    if (phase == 1 && ctx->n_sorted > 0) {
        unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
        for (int sx = 0; sx < ctx->narr; sx++)
            if ((src_mask >> sx) & 1u) want[dest_arr] |= 0xFFull << (8 * sx);
        if ((rc = prepare_lists(ctx, want, no_lists))) return rc;
    }
    b200sph_generic_args ga;
    memset(&ga, 0, sizeof(ga));
    for (int k = 0; k < (int)std::size(ga.f64); k++) ga.f64[k] = f64_ptr(ctx, B200SPH_X + k);
    for (int k = 0; k < (int)std::size(ga.f32); k++) ga.f32[k] = f32_ptr(ctx, B200SPH_P + k);
    for (int k = 0; k < (int)std::size(ga.u32); k++) ga.u32[k] = u32_ptr(ctx, B200SPH_GID + k);
    for (int k = 0; k < (int)std::size(ga.user); k++) ga.user[k] = f64_ptr(ctx, B200SPH_USER0 + k);
    ga.AB = ctx->AB; ga.stype = ctx->stype; ga.perm = ctx->perm;
    ga.cnt = ctx->cnt; ga.lst = ctx->lst; ga.capg = ctx->capg;
    ga.n = ctx->n_sorted;
    ga.cellx = (float)ctx->G.cell[0]; ga.celly = (float)ctx->G.cell[1]; ga.cellz = (float)ctx->G.cell[2];
    ga.k2 = (float)(ctx->radius_scale * ctx->radius_scale);
    ga.dest_type = dest_arr; ga.real_only = real_only; ga.phase = phase; ga.src_mask = src_mask;
    ga.t = t; ga.dt = dt;
    ga.doff = ctx->arr[dest_arr].off;
    ga.dlo = ranged ? ctx->dst_lo[dest_arr] : 0;
    ga.dhi = ranged && ctx->dst_hi[dest_arr] >= 0 ? ctx->dst_hi[dest_arr] : (int64_t)1 << 62;
    if (ctx->n_sorted > 0) {
        PhaseTimer pt(ctx, phase == 1 ? 1 : 2);
        const unsigned nb = (unsigned)cdiv(ctx->n_sorted, 128);
#ifdef B200SPH_HOST_EMULATION
        void (*fn)(b200sph_generic_args) = (void (*)(b200sph_generic_args))dlsym(ctx->gen_modules[module], kernel);
        if (!fn) return set_err(ctx, "generic_launch: no kernel '%s' in the module", kernel);
        emu::launch(nb, 128, emu::SEQ, [&] { fn(ga); });
#else
        void *fn = nullptr;
        int e = g_drv.ModuleGetFunction(&fn, ctx->gen_modules[module], kernel);
        if (e) return set_err(ctx, "generic_launch: no kernel '%s' in the module: %s", kernel, drv_err(e));
        void *params[1] = {&ga};
        e = g_drv.LaunchKernel(fn, nb, 1, 1, 128, 1, 1, 0, (void *)ctx->stream, params, nullptr);
        if (e) return set_err(ctx, "generic_launch: cuLaunchKernel(%s): %s", kernel, drv_err(e));
#endif
        ctx->stats.kernel_launches++;
    }
    // what was derived from the properties the bodies stored to is stale
    if (writes & 1) h_changed(ctx);
    if (writes & 2) state_changed(ctx), m_changed(ctx), ctx->spec_records = false;
    return 0;
}

// DensityCorrection's filter (density_filter.cuh).  Like generic_launch, a list consumer that
// writes a pool property between evaluations: the deferred initialize has copied the rho it
// overwrites (ensure_pool), the pending EOS calls are in the pool, and afterwards everything
// made from rho -- the packed records, the EOS speculatively applied to them -- is stale.
int b200sph_density_filter(b200sph_ctx *ctx, uint32_t array_mask, int mode, int kernel, int rhotmp_prop, int real_only)
{
    if (int rcc = require_confirmed(ctx, "density_filter")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (mode < B200SPH_DFILTER_SHEPARD || mode > B200SPH_DFILTER_MLS3D) return set_err(ctx, "density_filter: unknown mode %d", mode);
    if (kernel < 0 || kernel > 3) return set_err(ctx, "density_filter: unknown kernel id %d", kernel);
    if (kernel == B200SPH_KERNEL_WENDLAND_QUINTIC && ctx->dim == 1) return set_err(ctx, "WendlandQuintic: Dim 1 not supported");
    if (mode == B200SPH_DFILTER_MLS2D && ctx->dim != 2) return set_err(ctx, "density_filter: MLSFirstOrder2D needs dim = 2 (dim is %d)", ctx->dim);
    if (mode == B200SPH_DFILTER_MLS3D && ctx->dim != 3) return set_err(ctx, "density_filter: MLSFirstOrder3D needs dim = 3 (dim is %d)", ctx->dim);
    if (array_mask == 0 || array_mask >= (1u << ctx->narr)) return set_err(ctx, "density_filter: bad array mask 0x%x", array_mask);
    if (prop_kind(rhotmp_prop).group != GROUP_USER || !ctx->prop[rhotmp_prop])
        return set_err(ctx, "density_filter: rhotmp (property %d) is not a user property (b200sph_user_property)", rhotmp_prop);
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "density_filter runs on one GPU (no slab decomposition)");
    if (ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2] || mirror_any(ctx))
        return set_err(ctx, "density_filter: periodic and mirror domains are not supported");
    if (kernel_radius_scale(kernel) > ctx->radius_scale)
        return set_err(ctx, "density_filter: the filter kernel's radius scale (%g) exceeds the evaluation kernel's (%g), "
                            "which the neighbour lists are built for", kernel_radius_scale(kernel), ctx->radius_scale);
    if (!ctx->grid_valid) return set_err(ctx, "density_filter: the NNPS is stale (particles were pushed/resized); call nnps_update first");
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    if (ctx->n_sorted > 0) {
        // every filtered array is its own (only) source; the lists keep the union of what was asked
        unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
        for (int a = 0; a < ctx->narr; a++)
            if ((array_mask >> a) & 1u) want[a] |= 0xFFull << (8 * a);
        if ((rc = prepare_lists(ctx, want, "density_filter: the neighbour lists cannot index the particles"))) return rc;
        if ((rc = grow(ctx, ctx->dfilter_F, 2 * ctx->n_sorted, 2 * ctx->n_sorted))) return rc;
        PhaseTimer pt(ctx, 1);
        DensityFilterArgs fa;
        memset(&fa, 0, sizeof(fa));
        fa.AB = ctx->AB; fa.F = ctx->dfilter_F;
        fa.perm = ctx->perm; fa.cnt = ctx->cnt; fa.lst = ctx->lst; fa.stype = ctx->stype;
        fa.m = f64_ptr(ctx, B200SPH_M); fa.rho = f64_ptr(ctx, B200SPH_RHO); fa.rhotmp = f64_ptr(ctx, rhotmp_prop);
        fa.n = ctx->n_sorted; fa.capg = ctx->capg;
        fa.cellx = (float)ctx->G.cell[0]; fa.celly = (float)ctx->G.cell[1]; fa.cellz = (float)ctx->G.cell[2];
        const double kr = kernel_radius_scale(kernel);
        fa.k2 = (float)(kr * kr);
        fa.kfac = (float)kernel_fac(kernel, ctx->dim);
        fa.mask = array_mask;
        fa.real_only = real_only;
        k_dfilter_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(fa);
        LAUNCH_CHECK();
        const unsigned nb = (unsigned)cdiv(ctx->n_sorted, DFILTER_NT);
        rc = with_kernel_dim(ctx, kernel, ctx->dim, "density_filter", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if (mode == B200SPH_DFILTER_SHEPARD) k_density_filter<K, D, B200SPH_DFILTER_SHEPARD><<<nb, DFILTER_NT, 0, ctx->stream>>>(fa);
            else if constexpr (D == 2) k_density_filter<K, 2, B200SPH_DFILTER_MLS2D><<<nb, DFILTER_NT, 0, ctx->stream>>>(fa);
            else if constexpr (D == 3) k_density_filter<K, 3, B200SPH_DFILTER_MLS3D><<<nb, DFILTER_NT, 0, ctx->stream>>>(fa);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        ctx->stats.kernel_launches += 2;
    }
    // rho changed: the next evaluation packs its records (and applies its EOS) from it
    state_changed(ctx);
    ctx->spec_records = false;
    return 0;
}

// ---- particle shifting (shift_kernels.cuh) ---------------------------------------------------
// The checks, the invalidation rules and the records both entry points share.  Like
// density_filter, a list consumer that writes pool properties between evaluations: the deferred
// initialize has copied what it overwrites (ensure_pool: the write lands in the live x after the
// x / x0 rename), the pending EOS calls are in the pool, the lists cover the array's own pairs.
// The records are packed from the current pool.
static int shift_prepare(b200sph_ctx *ctx, const char *who, uint32_t array_mask, ShiftArgs &sa)
{
    if (int rcc = require_confirmed(ctx, who)) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (array_mask == 0 || array_mask >= (1u << ctx->narr)) return set_err(ctx, "%s: bad array mask 0x%x", who, array_mask);
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "%s runs on one GPU (no slab decomposition)", who);
    if (mirror_any(ctx)) return set_err(ctx, "%s: mirror domains are not supported", who);
    if (!ctx->grid_valid) return set_err(ctx, "%s: the NNPS is stale (particles were pushed, resized or moved); call nnps_update first", who);
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    memset(&sa, 0, sizeof(sa));
    if (ctx->n_sorted == 0) return 0;
    unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
    for (int a = 0; a < ctx->narr; a++)
        if ((array_mask >> a) & 1u) want[a] |= 0xFFull << (8 * a);
    char refusal[96];
    snprintf(refusal, sizeof(refusal), "%s: the neighbour lists cannot index the particles", who);
    if ((rc = prepare_lists(ctx, want, refusal))) return rc;
    const size_t n = (size_t)ctx->n_sorted, np = 3 * (size_t)ctx->pool_end;
    if ((rc = grow(ctx, ctx->shift_P, n, n)) || (rc = grow(ctx, ctx->shift_V, n, n)) ||
        (rc = grow(ctx, ctx->shift_dpos, np, np)) || (rc = grow(ctx, ctx->shift_dvel, np, np)) ||
        (rc = grow(ctx, ctx->shift_vmax, B200SPH_MAX_ARRAYS, B200SPH_MAX_ARRAYS)))
        return rc;
    sa.P = ctx->shift_P; sa.V = ctx->shift_V;
    sa.perm = ctx->perm; sa.cnt = ctx->cnt; sa.lst = ctx->lst; sa.skey = ctx->skey; sa.stype = ctx->stype;
    sa.x = f64_ptr(ctx, B200SPH_X); sa.y = f64_ptr(ctx, B200SPH_Y); sa.z = f64_ptr(ctx, B200SPH_Z);
    sa.u = f64_ptr(ctx, B200SPH_U); sa.v = f64_ptr(ctx, B200SPH_V); sa.w = f64_ptr(ctx, B200SPH_W);
    sa.h = f64_ptr(ctx, B200SPH_H); sa.m = f64_ptr(ctx, B200SPH_M); sa.rho = f64_ptr(ctx, B200SPH_RHO);
    sa.dpos = ctx->shift_dpos; sa.dvel = ctx->shift_dvel; sa.vmax = ctx->shift_vmax;
    sa.n = ctx->n_sorted; sa.capg = ctx->capg;
    sa.ncx = ctx->G.nc[0]; sa.ncy = ctx->G.nc[1]; sa.zorder = ctx->G.zorder;
    for (int d = 0; d < 3; d++) {
        sa.per[d] = ctx->G.periodic[d];
        sa.L[d] = ctx->dom_hi[d] - ctx->dom_lo[d];
    }
    sa.kr = ctx->radius_scale;
    sa.kfac = kernel_fac(ctx->kernel, ctx->dim);
    sa.mask = array_mask;
    k_shift_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(sa);
    LAUNCH_CHECK();
    return 0;
}

// ShiftPositions' shift Group: dpos of every real particle of the arrays in array_mask from the
// positions before the shift, then x += dpos.  The moved positions are judged by the next
// nnps_update's drift check against the build, like any other motion.
int b200sph_shift(b200sph_ctx *ctx, uint32_t array_mask, int kind, double dt, double coef, double hdx, int tensile,
                  double tensile_R, double tensile_n, int64_t *pairs)
{
    if (kind != B200SPH_SHIFT_SIMPLE && kind != B200SPH_SHIFT_FICKIAN) return set_err(ctx, "shift: unknown kind %d", kind);
    if (kind == B200SPH_SHIFT_FICKIAN && tensile && !(hdx > 0.0)) return set_err(ctx, "shift: FickianShift needs hdx > 0 (got %g)", hdx);
    ShiftArgs sa;
    int rc = shift_prepare(ctx, "shift", array_mask, sa);
    if (rc) return rc;
    if (ctx->n_sorted > 0) {
        PhaseTimer pt(ctx, 1);
        if ((rc = pairs_arm(ctx, pairs, &sa.pair_counter))) return rc;
        sa.dt = dt; sa.coef = coef; sa.hdx = hdx; sa.tensile = tensile; sa.tR = tensile_R; sa.tn = tensile_n;
        if (kind == B200SPH_SHIFT_SIMPLE) {
            // SimpleShift.py_initialize: vmax of each array, on the device
            CU(cudaMemsetAsync(ctx->shift_vmax, 0, sizeof(long long) * B200SPH_MAX_ARRAYS, ctx->stream));
            for (int a = 0; a < ctx->narr; a++)
                if (((array_mask >> a) & 1u) && ctx->arr[a].n > 0) {
                    k_shift_vmax<<<(unsigned)cdiv(ctx->arr[a].n, 256), 256, 0, ctx->stream>>>(
                        sa.u, sa.v, sa.w, ctx->arr[a].off, ctx->arr[a].n, ctx->shift_vmax + a);
                    LAUNCH_CHECK();
                }
        }
        const unsigned nb = (unsigned)cdiv(ctx->n_sorted, SHIFT_NT);
        rc = with_kernel_dim(ctx, "shift", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if (kind == B200SPH_SHIFT_SIMPLE) k_shift<K, D, B200SPH_SHIFT_SIMPLE><<<nb, SHIFT_NT, 0, ctx->stream>>>(sa);
            else k_shift<K, D, B200SPH_SHIFT_FICKIAN><<<nb, SHIFT_NT, 0, ctx->stream>>>(sa);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        k_shift_apply<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(sa, sa.dpos, sa.x, sa.y, sa.z);
        LAUNCH_CHECK();
        if ((rc = pairs_read(ctx, pairs))) return rc;
    } else if (pairs) {
        *pairs = 0;
    }
    ctx->shift_mask = array_mask;
    // x changed: the grid, the packed positions and the records made from them are stale
    particles_moved(ctx);
    ctx->spec_records = false;
    return 0;
}

// ShiftPositions' CorrectVelocities Group, after the neighbour search has seen the shifted
// positions: u += gradv . dpos with the dpos of the last b200sph_shift of these arrays.
int b200sph_correct_velocities(b200sph_ctx *ctx, uint32_t array_mask, int64_t *pairs)
{
    if (array_mask & ~ctx->shift_mask)
        return set_err(ctx, "correct_velocities: no shift of the arrays 0x%x since the particle set last changed (call b200sph_shift first)",
                       array_mask & ~ctx->shift_mask);
    ShiftArgs sa;
    int rc = shift_prepare(ctx, "correct_velocities", array_mask, sa);
    if (rc) return rc;
    if (ctx->n_sorted > 0) {
        PhaseTimer pt(ctx, 1);
        if ((rc = pairs_arm(ctx, pairs, &sa.pair_counter))) return rc;
        const unsigned nb = (unsigned)cdiv(ctx->n_sorted, SHIFT_NT);
        rc = with_kernel_dim(ctx, "correct_velocities", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            k_correct_velocities<K, D><<<nb, SHIFT_NT, 0, ctx->stream>>>(sa);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        k_shift_apply<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(sa, sa.dvel, sa.u, sa.v, sa.w);
        LAUNCH_CHECK();
        if ((rc = pairs_read(ctx, pairs))) return rc;
    } else if (pairs) {
        *pairs = 0;
    }
    // u, v, w changed: the next evaluation packs its records from them
    state_changed(ctx);
    ctx->spec_records = false;
    return 0;
}

// ---- Interpolator (interp_kernels.cuh) ----------------------------------------------------------
int b200sph_probe_create(b200sph_ctx *ctx, int64_t n, const double *x, const double *y, const double *z, double h)
{
    CU(cudaSetDevice(ctx->device));
    if (n < 0 || (n > 0 && (!x || !y || !z))) return set_err(ctx, "probe_create: bad points (n = %lld)", (long long)n);
    if (!(h > 0.0) || !std::isfinite(h)) return set_err(ctx, "probe_create: the probes' smoothing length must be > 0 (got %g)", h);
    b200sph_ctx::ProbeSet ps;
    ps.n = n;
    ps.h = h;
    if (n > 0) {
        if (int rc = grow(ctx, ps.xyz, 3 * n, 3 * n)) return rc;
        for (int d = 0; d < 3; d++)
            CU(cudaMemcpyAsync(ps.xyz + d * n, d == 0 ? x : (d == 1 ? y : z), 8 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    for (size_t i = 0; i < ctx->probes.size(); i++)
        if (ctx->probes[i].n < 0) {
            ctx->probes[i] = std::move(ps);
            return (int)i;
        }
    ctx->probes.push_back(std::move(ps));
    return (int)ctx->probes.size() - 1;
}

int b200sph_probe_release(b200sph_ctx *ctx, int id)
{
    if (id < 0 || id >= (int)ctx->probes.size() || ctx->probes[id].n < 0) return set_err(ctx, "probe_release: no probe set %d", id);
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    CU(ctx->probes[id].xyz.reset());
    ctx->probes[id].n = -1;   // a free slot
    return 0;
}

// A reader like pull_f64: the pending EOS calls are applied first, nothing the time loop caches
// is invalidated, and the only state it leaves behind is its own scratch.  It needs the build's
// sorted order to hold the current particle set, not its lists or a fresh grid: the stencil
// covers the drift since the build, measured in k_interp_pack.
int b200sph_interpolate(b200sph_ctx *ctx, int id, int method, int kernel, int dim, const int *props, uint32_t array_mask,
                        double *out)
{
    if (int rcc = require_confirmed(ctx, "interpolate")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (id < 0 || id >= (int)ctx->probes.size() || ctx->probes[id].n < 0) return set_err(ctx, "interpolate: no probe set %d", id);
    if (method < B200SPH_INTERP_SHEPARD || method > B200SPH_INTERP_ORDER1) return set_err(ctx, "interpolate: unknown method %d", method);
    if (kernel < 0 || kernel > 3) return set_err(ctx, "interpolate: unknown kernel id %d", kernel);
    if (dim < 1 || dim > 3) return set_err(ctx, "interpolate: dim must be 1, 2 or 3 (got %d)", dim);
    if (kernel == B200SPH_KERNEL_WENDLAND_QUINTIC && dim == 1) return set_err(ctx, "WendlandQuintic: Dim 1 not supported");
    if (array_mask == 0 || array_mask >= (1u << ctx->narr)) return set_err(ctx, "interpolate: bad array mask 0x%x", array_mask);
    if (!props) return set_err(ctx, "interpolate: no property ids");
    if (ctx->peer_box || ctx->comm_pending)
        return set_err(ctx, "interpolate runs on one GPU (no slab decomposition: a probe near a cut needs the other rank's particles)");
    InterpArgs ia;
    memset(&ia, 0, sizeof(ia));
    for (int a = 0; a < ctx->narr; a++) {
        const int p = props[a];
        if (p == -1 || !((array_mask >> a) & 1u)) continue;
        // a property without a buffer (nothing named it) is refused here, not allocated
        const PropType t = prop_kind(p).type;
        if (t == PROP_F64 && ctx->prop[p]) ia.fd[a] = f64_ptr(ctx, p);
        else if (t == PROP_F32 && ctx->prop[p]) ia.ff[a] = f32_ptr(ctx, p);
        else return set_err(ctx, "interpolate: property id %d (array %d) is not a floating-point property of the pool", p, a);
    }
    int64_t ntot = 0;
    for (int a = 0; a < ctx->narr; a++) ntot += ctx->arr[a].n;
    if (ctx->topo_dirty || ctx->n_sorted != ntot)
        return set_err(ctx, "interpolate: the particle set changed since the last neighbour-search build; call nnps_update first");
    const b200sph_ctx::ProbeSet &ps = ctx->probes[id];
    const double kr = kernel_radius_scale(kernel);
    // the stencil without the drift already visits a periodic cell twice
    for (int d = 0; d < 3; d++)
        if (ctx->G.periodic[d] && ntot > 0) {
            const int R = (int)std::ceil(kr * ps.h / ctx->G.cell[d]);
            if (2 * R + 1 > ctx->G.nc[d])
                return set_err(ctx, "interpolate: the stencil (%d cells) wraps onto itself along periodic axis %d (%d cells): "
                                    "the kernel's reach %g is too large for the box", 2 * R + 1, d, ctx->G.nc[d], kr * ps.h);
        }
    const size_t nout = (size_t)ps.n * (method == B200SPH_INTERP_ORDER1 ? 4 : 1);
    if (ps.n == 0) return 0;
    if (ntot == 0) {
        memset(out, 0, 8 * nout);
        return 0;
    }
    if ((rc = eos_flush(ctx))) return rc;
    const size_t ns = (size_t)ctx->n_sorted;
    if ((rc = grow(ctx, ctx->interp_Q, 2 * ns, 2 * ns)) || (rc = grow(ctx, ctx->interp_rho, ns, ns)) ||
        (rc = grow(ctx, ctx->interp_red, 8, 8)) || (rc = grow(ctx, ctx->interp_out, nout, nout)))
        return rc;
    {
        PhaseTimer pt(ctx, 2);
        ia.x = f64_ptr(ctx, B200SPH_X); ia.y = f64_ptr(ctx, B200SPH_Y); ia.z = f64_ptr(ctx, B200SPH_Z);
        ia.h = f64_ptr(ctx, B200SPH_H); ia.m = f64_ptr(ctx, B200SPH_M); ia.rho = f64_ptr(ctx, B200SPH_RHO);
        ia.perm = ctx->perm; ia.skey = ctx->skey; ia.cell_start = ctx->cell_start; ia.stype = ctx->stype;
        ia.n = ctx->n_sorted;
        ia.G = ctx->G;
        ia.Q = ctx->interp_Q; ia.rho_sph = ctx->interp_rho; ia.red = ctx->interp_red;
        ia.mask = array_mask;
        ia.px = ps.xyz; ia.py = ps.xyz + ps.n; ia.pz = ps.xyz + 2 * ps.n;
        ia.np = ps.n;
        ia.hp = (float)ps.h;
        ia.k = (float)kr;
        ia.kfac = (float)kernel_fac(kernel, dim);
        ia.method = method;
        ia.out = ctx->interp_out;
        CU(cudaMemsetAsync(ctx->interp_red, 0, 8 * sizeof(unsigned), ctx->stream));
        k_interp_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(ia);
        LAUNCH_CHECK();
        const unsigned nbp = (unsigned)cdiv(ps.n * 32, INTERP_NT);
        const unsigned nbd = (unsigned)cdiv(ctx->n_sorted * 32, INTERP_NT);
        rc = with_kernel_dim(ctx, kernel, dim, "interpolate", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if (method == B200SPH_INTERP_ORDER1) {
                k_interp_density<K, D><<<nbd, INTERP_NT, 0, ctx->stream>>>(ia);
                LAUNCH_CHECK();
                k_interp<K, D, true><<<nbp, INTERP_NT, 0, ctx->stream>>>(ia);
            } else {
                k_interp<K, D, false><<<nbp, INTERP_NT, 0, ctx->stream>>>(ia);
            }
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
    }
    unsigned wrapped = 0;
    CU(cudaMemcpyAsync(out, ctx->interp_out, 8 * nout, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&wrapped, ctx->interp_red + 4, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (wrapped)
        return set_err(ctx, "interpolate: the stencil wraps onto itself along a periodic axis: the kernel's reach plus the "
                            "drift since the last neighbour-search build spans the box; call nnps_update first");
    return 0;
}

int b200sph_set_dest_range(b200sph_ctx *ctx, int arr, int64_t start, int64_t stop)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "set_dest_range: bad array index %d", arr);
    if (start < 0 || stop < -1) return set_err(ctx, "set_dest_range: start >= 0 and stop >= 0 (or -1: no limit), got [%lld, %lld)", (long long)start, (long long)stop);
    if (!ctx->dst_ranged)
        for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) ctx->dst_lo[d] = 0, ctx->dst_hi[d] = -1;
    ctx->dst_lo[arr] = start;
    ctx->dst_hi[arr] = stop;
    ctx->dst_ranged = true;
    return 0;
}

// The 32-byte records (k_pair_list_r32) serve a list-walking pass of the WCSPH scheme's Group
// (not ranged) when every array has a pending Tait EOS with gamma = 7 and the same rho0, c0
// and pressure offset, h and m are the same for every particle, and there are no ghosts (the
// slab halo and the mirror images write 48-byte records).  B200SPH_RECORDS=48 keeps the
// 48-byte layout everywhere.
static double eos_offset(const EosTab &E, int a) { return E.hg[a] ? 0.0 : E.p0[a]; }
static Rec32Eos rec32_eos(const EosTab &E, int a)
{
    const double rho0 = E.rho0[a], B = rho0 * E.c0[a] * E.c0[a] / 7.0, kB = B / (rho0 * rho0);
    return Rec32Eos{rho0, B, eos_offset(E, a), {(float)kB, (float)(7.0 * kB), (float)(21.0 * kB), (float)(35.0 * kB)},
                    (float)(eos_offset(E, a) / (rho0 * rho0))};
}
static int records32(b200sph_ctx *ctx, const bool wcsph_list_pass, bool *yes, int *eos_arr)
{
    *yes = false;
    if (ctx->rec48_forced || !wcsph_list_pass || !ctx->eos_any || mirror_any(ctx) || ctx->peer_box || ctx->comm_pending)
        return 0;
    const EosTab &E = ctx->eos_pending;
    int &first = *eos_arr;
    first = -1;
    for (int a = 0; a < ctx->narr; a++) {
        if (ctx->arr[a].n != ctx->arr[a].n_real) return 0;
        if (ctx->arr[a].n == 0) continue;
        if (!E.on[a] || E.gamma[a] != 7.0) return 0;
        if (first < 0) first = a;
        else if (E.rho0[a] != E.rho0[first] || E.c0[a] != E.c0[first] || eos_offset(E, a) != eos_offset(E, first)) return 0;
    }
    if (first < 0) return 0;
    if (int rc = hm_uniformity(ctx)) return rc;
    *yes = !std::isnan(ctx->h_uniform) && !std::isnan(ctx->m_uniform);
    return 0;
}

static bool can_fuse_stage(const b200sph_ctx *ctx, int arr);
int b200sph_pair_pass(b200sph_ctx *ctx, const b200sph_pair_program *prog, int64_t *pairs_out)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, false, true);   // a halo in flight is waited for below, as late as possible
    if (rc) return rc;
    if (!ctx->grid_valid) return set_err(ctx, "pair_pass: the NNPS is stale (particles were pushed/resized); call nnps_update first");
    if (ctx->spec_records && ctx->state_packed) {
        // records packed by the fused stage kernel: valid only if this evaluation issued
        // exactly the equation-of-state calls that were applied speculatively
        unsigned want = 0, pending = 0;
        for (int a = 0; a < ctx->narr; a++) {
            if (ctx->eos_last_valid && ctx->eos_last.on[a]) want |= 1u << a;
            if (ctx->eos_any && ctx->eos_pending.on[a]) pending |= 1u << a;
        }
        if (pending != want || ctx->spec_confirmed != want) state_changed(ctx);
    }
    ctx->spec_records = false;
    ctx->spec_confirmed = 0;
    ctx->dt_reduced = false;   // this pass writes new dt_cfl / dt_force
    if (ctx->eos_any) {
        ctx->eos_last = ctx->eos_pending;
        ctx->eos_last_valid = true;
    } else {
        ctx->eos_last_valid = false;
    }
    const bool use_lists = ctx->n_sorted > 0 && lists_usable(ctx, ctx->n_sorted);
    const bool ranged = ctx->dst_ranged;
    ctx->dst_ranged = false;
    if (ranged && !use_lists && ctx->n_sorted > 0)
        return set_err(ctx, "pair_pass: destination ranges (Group start_idx / stop_idx) need the neighbour-list path");
    // the WCSPH scheme's Group (continuity + momentum + XSPH, no tensile correction) has a
    // leaner kernel variant, and may have 32-byte records
    unsigned prog_bits = 0;
    for (int d = 0; d < ctx->narr; d++)
        for (int sx = 0; sx < ctx->narr; sx++) prog_bits |= prog->eqmask[d][sx];
    const bool wcsph_only = !(prog_bits & ~(unsigned)PAIR_EQS_WCSPH) && !prog->tensile_correction;
    // SummationDensity stores rho: a deferred initialize must have copied it before, and a
    // pending half step formed it
    const bool writes_rho = (prog_bits & B200SPH_EQ_SUMMATION_DENSITY) != 0;
    if (writes_rho && (rc = materialise_pending(ctx))) return rc;
    bool r32 = false;
    int ea = -1;
    if ((rc = records32(ctx, use_lists && !ranged && wcsph_only, &r32, &ea))) return rc;
    const EosTab E32 = ctx->eos_pending;   // (packing the state retires the pending calls)
    // records packed with another EOS (rho0, c0 or offset; by k_pack_rec32 or, speculatively,
    // by k_stage_pack) are stale even when the same EOS calls are pending
    const Rec32Eos key = r32 ? rec32_eos(E32, ea) : Rec32Eos{};
    if (r32 != ctx->rec32 || (r32 && key != ctx->rec32_eos)) {
        ctx->rec32 = r32;
        ctx->rec32_eos = key;
        state_changed(ctx);
    }
    if (!r32 && (rc = ab_positions(ctx))) return rc;
    // the (destination, source) type pairs this Group has equations for; lists that were
    // filtered with a narrower set are rebuilt with the union
    unsigned long long want[B200SPH_MAX_ARRAYS];
    for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) {
        want[d] = 0;
        for (int sx = 0; sx < B200SPH_MAX_ARRAYS; sx++)
            if (d < ctx->narr && sx < ctx->narr && prog->eqmask[d][sx]) want[d] |= 0xFFull << (8 * sx);
    }
    // the peer protocol's refresh is still in flight and every record a ghost-free CTA
    // reads is in place: those CTAs go first, the main stream waits for the halo only then
    const bool overlap = ctx->comm_pending && use_lists && ctx->lists_valid && lists_cover(ctx, want) && ctx->chunks_valid &&
                         ctx->state_packed && ctx->n_chunk_interior > 0 && !pairs_out && !ranged;
    if (!overlap && (rc = sync_comm(ctx))) return rc;
    if (!ctx->state_packed) {
        if ((rc = pack_state(ctx))) return rc;
    } else if (!overlap) {
        // the records have the calls; the pool's rho / p / cs get them now or, when the next
        // stage can be the fused kernel and this pass leaves rho alone, in that kernel
        if (ctx->eos_any && !ctx->eos_pool_any && !writes_rho && !ctx->peer_box && can_fuse_stage(ctx, -1)) {
            ctx->eos_pool = ctx->eos_pending;
            ctx->eos_pool_any = true;
            memset(ctx->eos_pending.on, 0, sizeof(ctx->eos_pending.on));
            ctx->eos_any = false;
        } else if ((ctx->eos_any || writes_rho) && (rc = eos_flush(ctx))) {
            return rc;
        }
    }
    if (!use_lists && (ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2]))
        return set_err(ctx, "periodic domains need the neighbour-list path (B200SPH_PAIR_KERNEL=list, < 2^26 particles)");
    if (use_lists && (rc = prepare_lists(ctx, want, "pair_pass: the lists cannot index the particles"))) return rc;
    // the accelerations of the evaluation before a pending half step are still needed: this pass
    // writes into the spare set, or (another pair kernel) the half step is formed now
    const unsigned acc_w = acc_writes(ctx, prog, r32);
    if (ctx->half_pending && !ctx->acc_swapped && acc_w) {
        if (r32 && use_lists) rc = acc_swap(ctx, acc_w);
        else rc = half_materialise(ctx);
        if (rc) return rc;
    }
    ctx->acc_differ |= acc_w;
    PhaseTimer pt(ctx, 1);

    PairArgs pa;
    memset(&pa, 0, sizeof(pa));
    pa.A = ctx->A; pa.B = ctx->B; pa.C = ctx->C; pa.AB = ctx->AB;
    pa.cell_start = ctx->cell_start; pa.skey = ctx->skey; pa.perm = ctx->perm;
    pa.arho = f32_ptr(ctx, B200SPH_ARHO);
    pa.au = f32_ptr(ctx, B200SPH_AU); pa.av = f32_ptr(ctx, B200SPH_AV); pa.aw = f32_ptr(ctx, B200SPH_AW);
    pa.ax = f32_ptr(ctx, B200SPH_AX); pa.ay = f32_ptr(ctx, B200SPH_AY); pa.az = f32_ptr(ctx, B200SPH_AZ);
    pa.dt_cfl = f32_ptr(ctx, B200SPH_DT_CFL); pa.dt_force = f32_ptr(ctx, B200SPH_DT_FORCE);
    pa.rho = f64_ptr(ctx, B200SPH_RHO);
    pa.n = ctx->n_sorted;
    pa.ncx = ctx->G.nc[0]; pa.ncy = ctx->G.nc[1]; pa.ncz = ctx->G.nc[2];
    pa.zorder = ctx->G.zorder;
    pa.cellx = (float)ctx->G.cell[0]; pa.celly = (float)ctx->G.cell[1]; pa.cellz = (float)ctx->G.cell[2];
    pa.k2 = (float)(ctx->radius_scale * ctx->radius_scale);
    pa.kfac = (float)kernel_fac(ctx->kernel, ctx->dim);
    pa.deltap = (float)kernel_deltap(ctx->kernel);
    bool sumdens = false;
    for (int d = 0; d < B200SPH_MAX_ARRAYS; d++) {
        unsigned long long m = 0;
        for (int s = 0; s < B200SPH_MAX_ARRAYS; s++) {
            const uint32_t b = (d < ctx->narr && s < ctx->narr) ? prog->eqmask[d][s] : 0u;
            if (b > 0xFFu) return set_err(ctx, "pair_pass: unknown equation bits 0x%x", b);
            m |= (unsigned long long)b << (8 * s);
            if (b & B200SPH_EQ_SUMMATION_DENSITY) sumdens = true;
        }
        pa.emask[d] = m;
    }
    pa.c0 = (float)prog->c0; pa.alpha = (float)prog->alpha; pa.beta = (float)prog->beta;
    pa.gx = (float)prog->gx; pa.gy = (float)prog->gy; pa.gz = (float)prog->gz;
    pa.eps_xsph = (float)prog->eps_xsph;
    pa.nu4 = (float)(4.0 * prog->nu); pa.eta = (float)prog->eta;
    pa.tensile = prog->tensile_correction;
    pa.real_only = prog->real_only;
    PairR32 pc;
    memset(&pc, 0, sizeof(pc));
    if (r32) {
        const double rho0 = E32.rho0[ea], c0 = E32.c0[ea];
        pa.R = ctx->R;
        pa.h = (float)ctx->h_uniform;        // the float every A record holds
        pa.m = (float)ctx->m_uniform;
        pa.rho0 = (float)rho0;
        pa.hrho0 = (float)(0.5 * rho0);
        pa.ac0 = (float)(-0.5 * prog->alpha * c0);
        const double h = pa.h, h1 = 1.0 / h, fac = kernel_fac(ctx->kernel, ctx->dim) * pow(h1, ctx->dim);
        pc.h1 = (float)h1;
        pc.gfac = (float)(fac * h1);
        pc.wfac = (float)fac;
        pc.eta2 = (float)(0.01 * h * h);
        for (int d = 0; d < ctx->narr; d++)
            for (int s = 0; s < ctx->narr; s++) {
                const uint32_t b = prog->eqmask[d][s];
                pc.esel[d] |= (b ? 1u << (ESEL_ANY + s) : 0u) | ((b & B200SPH_EQ_CONTINUITY) ? 1u << (ESEL_CONTINUITY + s) : 0u) |
                              ((b & B200SPH_EQ_MOMENTUM) ? 1u << (ESEL_MOMENTUM + s) : 0u) |
                              ((b & B200SPH_EQ_XSPH) ? 1u << (ESEL_XSPH + s) : 0u);
            }
    }
    if (ranged)
        for (int d = 0; d < ctx->narr; d++) {
            pa.doff[d] = ctx->arr[d].off;
            pa.dlo[d] = ctx->dst_lo[d];
            pa.dhi[d] = ctx->dst_hi[d] < 0 ? (int64_t)1 << 62 : ctx->dst_hi[d];
        }
    if ((rc = pairs_arm(ctx, pairs_out, &pa.pair_counter))) return rc;
    if (use_lists) {
        // phase 0: every CTA, or (overlap) the ghost-free CTAs on the main stream; phase 1: the
        // others on the COMMUNICATION stream, in order behind the halo scatter -- the two
        // launches run side by side, the boundary CTAs (higher stream priority) take the SM
        // slots the interior CTAs free, and there is one tail instead of two.  The main
        // stream joins when the next entry point needs the results (sync_comm).
        for (int phase = 0; phase < (overlap ? 2 : 1); phase++) {
            const uint32_t *ids = !overlap ? nullptr : (phase == 0 ? ctx->chunk_interior.p : ctx->chunk_boundary.p);
            const unsigned nb = (unsigned)(!overlap ? cdiv(ctx->n_sorted, LIST_NT) : (phase == 0 ? ctx->n_chunk_interior : ctx->n_chunk_boundary));
            cudaStream_t lst_stream = ctx->stream;
            if (phase == 1) {
                lst_stream = ctx->comm_stream;
                if ((rc = eos_flush(ctx, ctx->comm_stream))) return rc;   // pool side of the speculated EOS, ghosts included
                ctx->n_overlapped++;
            }
            if (nb == 0) continue;
            rc = with_kernel_dim(ctx, "pair_pass", [&](auto kc, auto dc) {
                constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
                if (r32) k_pair_list_r32<K, D><<<nb, LIST_NT, 0, lst_stream>>>(pa, pc, ctx->cnt, ctx->lst, ctx->capg);
                else if (ranged) k_pair_list<K, D, 6, PAIR_EQS_ALL, true><<<nb, LIST_NT, 0, lst_stream>>>(pa, ctx->cnt, ctx->lst, ctx->capg, ids);
                else if (wcsph_only) k_pair_list<K, D, 7, PAIR_EQS_WCSPH><<<nb, LIST_NT, 0, lst_stream>>>(pa, ctx->cnt, ctx->lst, ctx->capg, ids);
                else k_pair_list<K, D, 7, PAIR_EQS_ALL><<<nb, LIST_NT, 0, lst_stream>>>(pa, ctx->cnt, ctx->lst, ctx->capg, ids);
                LAUNCH_CHECK();
                return 0;
            });
            if (rc) return rc;
        }
        if (overlap) {   // the join point moves behind the boundary launch
            CU(cudaEventRecord(ctx->ev_join, ctx->comm_stream));
            ctx->comm_pending = true;
            if (ctx->profiling && ctx->halo_ev_fork && ctx->halo_ev_chain) {
                cudaEvent_t e_end = nullptr;
                if (!ctx->ev_pool.empty()) { e_end = ctx->ev_pool.back(); ctx->ev_pool.pop_back(); }
                else CU(cudaEventCreate(&e_end));
                CU(cudaEventRecord(e_end, ctx->comm_stream));
                ctx->halo_pending.push_back({ctx->halo_ev_fork, ctx->halo_ev_chain, e_end, ctx->halo_ev_sent, ctx->halo_ev_reduced});
                ctx->halo_ev_fork = ctx->halo_ev_chain = ctx->halo_ev_sent = ctx->halo_ev_reduced = nullptr;
            }
        }
        ctx->stats.pair_launches++;
        if (r32) ctx->n_pair_r32++;
    } else if (ctx->n_sorted > 0) {
        const unsigned nb = (unsigned)cdiv(ctx->n_sorted, PAIR_WARPS * PAIR_CHUNK);
        rc = with_kernel_dim(ctx, "pair_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            k_pair<K, D><<<nb, PAIR_WARPS * 32, 0, ctx->stream>>>(pa);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        ctx->stats.pair_launches++;
    }
    if ((rc = pairs_read(ctx, pairs_out))) return rc;
    if (sumdens) state_changed(ctx);  // rho changed
    return 0;
}

int b200sph_tvf_pass(b200sph_ctx *ctx, const b200sph_tvf_program *prog, int64_t *pairs_out)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (!ctx->grid_valid) return set_err(ctx, "tvf_pass: the NNPS is stale (particles were pushed/resized); call nnps_update first");
    if (!(prog->passes & 7)) return set_err(ctx, "tvf_pass: passes must select group 1, the average-pressure group and/or group 2");
    if (prog->eqbits > 255u) return set_err(ctx, "tvf_pass: unknown equation bits 0x%x", prog->eqbits);
    const bool ext = (prog->eqbits & (B200SPH_TVF_MOM | B200SPH_TVF_XSPH)) != 0;
    if (ext && (prog->eqbits & (B200SPH_TVF_PGRAD | B200SPH_TVF_ASTRESS)))
        return set_err(ctx, "tvf_pass: equations of the internal-flow (transport velocity) and of the external-flow branch in one Group");
    if (prog->clamp_p && !prog->solid_mask) return set_err(ctx, "tvf_pass: ClampWallPressure without a solid wall");
    if (prog->fluid_mask == 0 || prog->fluid_mask >= (1u << ctx->narr)) return set_err(ctx, "tvf_pass: bad fluid mask 0x%x", prog->fluid_mask);
    const unsigned solid_mask = prog->solid_mask;
    if (solid_mask >= (1u << ctx->narr) || (solid_mask & prog->fluid_mask))
        return set_err(ctx, "tvf_pass: bad solid mask 0x%x (fluids 0x%x)", solid_mask, prog->fluid_mask);
    if ((prog->eqbits & B200SPH_TVF_NOSLIP) && !solid_mask) return set_err(ctx, "tvf_pass: SolidWallNoSlipBC without a solid wall");
    if ((prog->passes & 4) && ext) return set_err(ctx, "tvf_pass: the external-flow branch has no average pressure");
    if ((prog->passes & 4) && !solid_mask) return set_err(ctx, "tvf_pass: the average pressure has a Group of its own only with solid walls");
    if ((prog->passes & 1) && solid_mask && prog->bql)
        return set_err(ctx, "tvf_pass: with solid walls the average pressure is computed after the wall pressure (passes bit 2), not in group 1");
    if (solid_mask && (ctx->peer_box || ctx->comm_pending)) return set_err(ctx, "tvf_pass: EDAC with solid walls runs on one GPU");
    if (ctx->n_sorted == 0) return 0;
    if ((rc = ab_positions(ctx))) return rc;
    // (these passes take unfiltered lists)
    if ((rc = prepare_lists(ctx, nullptr, "tvf_pass: the EDAC kernels need the neighbour-list path (B200SPH_PAIR_KERNEL=list, < 2^26 particles)")))
        return rc;
    // timing slots: pack + group 1 count as "other", group 2 (the dominant kernel) as "pair"
    PhaseTimer pt(ctx, 2);
    const unsigned nbp = (unsigned)cdiv(ctx->n_sorted, 256);
    k_pack_tvf<<<nbp, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_U), f64_ptr(ctx, B200SPH_V), f64_ptr(ctx, B200SPH_W), f64_ptr(ctx, B200SPH_M),
                                             f64_ptr(ctx, B200SPH_UHAT), f64_ptr(ctx, B200SPH_VHAT),
                                             f64_ptr(ctx, B200SPH_WHAT), f64_ptr(ctx, B200SPH_PF),
                                             f32_ptr(ctx, B200SPH_PAVG), ctx->ptype, ctx->perm, ctx->n_sorted,
                                             ctx->B, ctx->AB, ctx->C, ctx->Dv, ctx->PT, f64_ptr(ctx, B200SPH_RHO), solid_mask);
    LAUNCH_CHECK();
    state_changed(ctx);   // B / C no longer hold the WCSPH records

    TvfArgs ta;
    memset(&ta, 0, sizeof(ta));
    ta.AB = ctx->AB; ta.C2 = ctx->C; ta.Dv = ctx->Dv; ta.PT = ctx->PT; ta.perm = ctx->perm;
    ta.rho = f64_ptr(ctx, B200SPH_RHO);
    ta.V = f32_ptr(ctx, B200SPH_VOL); ta.pavg = f32_ptr(ctx, B200SPH_PAVG);
    ta.au = f32_ptr(ctx, B200SPH_AU); ta.av = f32_ptr(ctx, B200SPH_AV); ta.aw = f32_ptr(ctx, B200SPH_AW);
    ta.auhat = f32_ptr(ctx, B200SPH_AUHAT); ta.avhat = f32_ptr(ctx, B200SPH_AVHAT);
    ta.awhat = f32_ptr(ctx, B200SPH_AWHAT); ta.ap = f32_ptr(ctx, B200SPH_AP);
    ta.n = ctx->n_sorted;
    ta.cellx = (float)ctx->G.cell[0]; ta.celly = (float)ctx->G.cell[1]; ta.cellz = (float)ctx->G.cell[2];
    ta.k2 = (float)(ctx->radius_scale * ctx->radius_scale);
    ta.kfac = (float)kernel_fac(ctx->kernel, ctx->dim);
    ta.fluid_mask = prog->fluid_mask;
    ta.solid_mask = solid_mask;
    ta.src_mask = prog->fluid_mask | solid_mask;
    ta.eqbits = prog->eqbits;
    ta.bql = prog->bql;
    ta.wgx = (float)prog->gx; ta.wgy = (float)prog->gy; ta.wgz = (float)prog->gz;
    ta.eps_xsph = (float)prog->eps_xsph;
    ta.clamp_p = prog->clamp_p;
    ta.ax = f32_ptr(ctx, B200SPH_AX); ta.ay = f32_ptr(ctx, B200SPH_AY); ta.az = f32_ptr(ctx, B200SPH_AZ);
    ta.p32 = f32_ptr(ctx, B200SPH_P);
    ta.ug = f64_ptr(ctx, B200SPH_UHAT); ta.vg = f64_ptr(ctx, B200SPH_VHAT);
    ta.wg = f64_ptr(ctx, B200SPH_WHAT);
    ta.pb = (float)prog->pb; ta.nu = (float)prog->nu; ta.edac_nu = (float)prog->edac_nu;
    ta.c0 = (float)prog->c0; ta.alpha = (float)prog->alpha;
    double damp = 1.0;   // wc/edac.py:483-488
    if (prog->t < prog->tdamp) damp = 0.5 * (std::sin((-0.5 + prog->t / prog->tdamp) * 3.14159265358979323846) + 1.0);
    ta.gx = (float)(prog->gx * damp); ta.gy = (float)(prog->gy * damp); ta.gz = (float)(prog->gz * damp);
    if ((rc = pairs_arm(ctx, pairs_out, &ta.pair_counter))) return rc;
    const unsigned nb = (unsigned)cdiv(ctx->n_sorted, LIST_NT);
    // stages: 1 group 1 (fluids), 2 group 1 (wall arrays), 3 the average-pressure group, 4 group 2
    for (int stage = 1; stage <= 4; stage++) {
        const int pass = stage == 4 ? 2 : 1;
        if (stage == 4) pt.to(1);
        if (stage == 1 && !(prog->passes & 1)) continue;
        if (stage == 2 && !((prog->passes & 1) && solid_mask)) continue;
        if (stage == 3 && !(prog->passes & 4)) continue;
        if (stage == 4 && !(prog->passes & 2)) continue;
        ta.avg_only = stage == 3 ? 1 : 0;
        if (stage == 3) ta.bql = 1;
        rc = with_kernel_dim(ctx, "tvf_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if (stage == 2) k_tvf_wall<K, D><<<nb, LIST_NT, 0, ctx->stream>>>(ta, ctx->cnt, ctx->lst, ctx->capg);
            else if (pass == 1) k_tvf_pass1<K, D><<<nb, LIST_NT, 0, ctx->stream>>>(ta, ctx->cnt, ctx->lst, ctx->capg);
            else if (ext) k_tvf_pass2<K, D, true, true><<<nb, LIST_NT, 0, ctx->stream>>>(ta, ctx->cnt, ctx->lst, ctx->capg);
            else if (solid_mask) k_tvf_pass2<K, D, true><<<nb, LIST_NT, 0, ctx->stream>>>(ta, ctx->cnt, ctx->lst, ctx->capg);
            else k_tvf_pass2<K, D><<<nb, LIST_NT, 0, ctx->stream>>>(ta, ctx->cnt, ctx->lst, ctx->capg);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        if (stage == 3) ta.bql = prog->bql;
        if (pass == 2) ctx->stats.pair_launches++;
    }
    pt.stop();
    return pairs_read(ctx, pairs_out);
}

int b200sph_solid_pass(b200sph_ctx *ctx, const b200sph_solid_program *prog, int64_t *pairs_out)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if ((rc = ensure_prop(ctx, B200SPH_S00))) return rc;
    if (!ctx->grid_valid) return set_err(ctx, "solid_pass: the NNPS is stale (particles were pushed/resized); call nnps_update first");
    if (!(prog->passes & 3)) return set_err(ctx, "solid_pass: passes must select group 1 and/or group 2");
    if (prog->elastic_mask == 0 || prog->elastic_mask >= (1u << ctx->narr)) return set_err(ctx, "solid_pass: bad elastic mask 0x%x", prog->elastic_mask);
    if (ctx->n_sorted == 0) return 0;
    if ((rc = ab_positions(ctx))) return rc;
    // (these passes take unfiltered lists)
    if ((rc = prepare_lists(ctx, nullptr, "solid_pass: the elastic-dynamics kernels need the neighbour-list path"))) return rc;
    SolidArgs sa;
    memset(&sa, 0, sizeof(sa));
    sa.AB = ctx->AB; sa.C3 = ctx->C; sa.T01 = ctx->T01; sa.T2R = ctx->T2R; sa.R2 = ctx->R2; sa.perm = ctx->perm;
    sa.rho = f64_ptr(ctx, B200SPH_RHO);
    for (int k = 0; k < 6; k++) {
        sa.s[k] = f64_ptr(ctx, B200SPH_S00 + k);
        sa.r[k] = f32_ptr(ctx, B200SPH_R00 + k);
        sa.as[k] = f32_ptr(ctx, B200SPH_AS00 + k);
    }
    for (int k = 0; k < 9; k++) sa.vg[k] = f32_ptr(ctx, B200SPH_V00 + k);
    sa.p = f32_ptr(ctx, B200SPH_P);
    sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    sa.au = f32_ptr(ctx, B200SPH_AU); sa.av = f32_ptr(ctx, B200SPH_AV); sa.aw = f32_ptr(ctx, B200SPH_AW);
    sa.ax = f32_ptr(ctx, B200SPH_AX); sa.ay = f32_ptr(ctx, B200SPH_AY); sa.az = f32_ptr(ctx, B200SPH_AZ);
    sa.n = ctx->n_sorted;
    sa.cellx = (float)ctx->G.cell[0]; sa.celly = (float)ctx->G.cell[1]; sa.cellz = (float)ctx->G.cell[2];
    sa.k2 = (float)(ctx->radius_scale * ctx->radius_scale);
    sa.kfac = (float)kernel_fac(ctx->kernel, ctx->dim);
    sa.elastic_mask = prog->elastic_mask;
    sa.source_mask = prog->source_mask ? prog->source_mask : prog->elastic_mask;
    if ((sa.source_mask & sa.elastic_mask) != sa.elastic_mask) return set_err(ctx, "solid_pass: every elastic array must be a source");
    sa.grad3d = prog->grad3d;
    sa.ghost_group1 = prog->ghost_group1;
    sa.eps = (float)prog->eps; sa.alpha = (float)prog->alpha; sa.beta = (float)prog->beta; sa.eps_xsph = (float)prog->eps_xsph;
    for (int a = 0; a < B200SPH_MAX_ARRAYS; a++) {
        sa.c0_ref[a] = prog->c0_ref[a]; sa.rho_ref[a] = prog->rho_ref[a]; sa.G[a] = prog->G[a];
        sa.wdeltap[a] = (float)prog->wdeltap[a]; sa.nexp[a] = (float)prog->n[a];
    }
    if ((rc = pairs_arm(ctx, pairs_out, &sa.pair_counter))) return rc;
    PhaseTimer pt(ctx, 2);
    if (prog->passes & 1) {
        // group 2 alone reuses the records the last group 1 left behind
        k_pack_solid<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(
            f64_ptr(ctx, B200SPH_U), f64_ptr(ctx, B200SPH_V), f64_ptr(ctx, B200SPH_W), f64_ptr(ctx, B200SPH_M), f64_ptr(ctx, B200SPH_RHO),
            f32_ptr(ctx, B200SPH_P), f32_ptr(ctx, B200SPH_CS), ctx->ptype, ctx->perm, ctx->n_sorted, ctx->B, ctx->AB, ctx->C);
        LAUNCH_CHECK();
        state_changed(ctx);   // B / C no longer hold the WCSPH records
    }
    const unsigned nb = (unsigned)cdiv(ctx->n_sorted, LIST_NT);
    for (int pass = 1; pass <= 2; pass++) {
        if (pass == 2) pt.to(1);
        if (!(prog->passes & pass)) continue;
        rc = with_kernel_dim(ctx, "solid_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if (pass == 1) k_solid_pass1<K, D><<<nb, LIST_NT, 0, ctx->stream>>>(sa, ctx->cnt, ctx->lst, ctx->capg);
            else k_solid_pass2<K, D><<<nb, LIST_NT, 0, ctx->stream>>>(sa, ctx->cnt, ctx->lst, ctx->capg);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
        if (pass == 2) ctx->stats.pair_launches++;
    }
    pt.stop();
    return pairs_read(ctx, pairs_out);
}

static int ensure_tc(b200sph_ctx *ctx);
// what every stage entry point (WCSPHStep, WCSPHTVDRK3Step, the EDAC steppers, SolidMechStep)
// checks and prepares before it fills its arguments; `last` is the stepper's last stage
static int stage_begin(b200sph_ctx *ctx, const char *who, int arr, int which, bool devdt, int last = 2, bool keep_init = false)
{
    if (int rcc = require_confirmed(ctx, who)) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, true, keep_init);
    if (rc) return rc;
    if (arr >= ctx->narr) return set_err(ctx, "%s: bad array %d", who, arr);
    if (last == 3 && (which < 0 || which > 3))
        return set_err(ctx, "%s: which must be 0 (initialize), 1 (stage1), 2 (stage2) or 3 (stage3)", who);
    if (which < 0 || which > last) return set_err(ctx, "%s: which must be 0 (initialize), 1 (stage1) or 2 (stage2)", who);
    if (devdt && (rc = ensure_tc(ctx))) return rc;
    return 0;
}

static int stage_solid_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt)
{
    int rc = stage_begin(ctx, "stage_solid", arr, which, devdt);
    if (rc || (rc = ensure_prop(ctx, B200SPH_S00))) return rc;
    PhaseTimer pt(ctx, 2);
    StageSolidArgs sa;
    stage_args(ctx, sa, arr, which, dt, devdt);
    sa.rho = f64_ptr(ctx, B200SPH_RHO); sa.rho0 = f64_ptr(ctx, B200SPH_RHO0); sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    for (int k = 0; k < 6; k++) {
        sa.s[k] = f64_ptr(ctx, B200SPH_S00 + k);
        sa.s0[k] = f64_ptr(ctx, B200SPH_S000 + k);
        sa.as[k] = f32_ptr(ctx, B200SPH_AS00 + k);
    }
    if (ctx->pool_end > 0) {
        k_stage_solid<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    if (which != 0) particles_moved(ctx);
    return 0;
}
int b200sph_stage_solid(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_solid_impl(ctx, arr, which, dt, false); }
int b200sph_stage_solid_dev(b200sph_ctx *ctx, int arr, int which) { return stage_solid_impl(ctx, arr, which, 0.0, true); }

static int stage_tvf_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt, int ext = 0)
{
    int rc = stage_begin(ctx, "stage_tvf", arr, which, devdt);
    if (rc) return rc;
    PhaseTimer pt(ctx, 2);
    StageTvfArgs sa;
    stage_args(ctx, sa, arr, which, dt, devdt);
    sa.uh = f64_ptr(ctx, B200SPH_UHAT); sa.vh = f64_ptr(ctx, B200SPH_VHAT); sa.wh = f64_ptr(ctx, B200SPH_WHAT);
    sa.pf = f64_ptr(ctx, B200SPH_PF); sa.pf0 = f64_ptr(ctx, B200SPH_PF0);
    sa.auh = f32_ptr(ctx, B200SPH_AUHAT); sa.avh = f32_ptr(ctx, B200SPH_AVHAT);
    sa.awh = f32_ptr(ctx, B200SPH_AWHAT); sa.ap = f32_ptr(ctx, B200SPH_AP);
    sa.ext = ext;
    if (ctx->pool_end > 0) {
        k_stage_tvf<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    if (which != 0) particles_moved(ctx);
    return 0;
}
int b200sph_stage_tvf(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_tvf_impl(ctx, arr, which, dt, false); }
int b200sph_stage_tvf_dev(b200sph_ctx *ctx, int arr, int which) { return stage_tvf_impl(ctx, arr, which, 0.0, true); }
int b200sph_stage_edac(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_tvf_impl(ctx, arr, which, dt, false, 1); }
int b200sph_stage_edac_dev(b200sph_ctx *ctx, int arr, int which) { return stage_tvf_impl(ctx, arr, which, 0.0, true, 1); }

static int ensure_tc(b200sph_ctx *ctx)
{
    if (ctx->tc) return 0;
    if (int rc = grow(ctx, ctx->tc_own, 8, 8)) return rc;
    ctx->tc = ctx->tc_own;
    const double init[8] = {0.0, 0.0, 1e20, -1.0, 0.0, 0.0, 0.0, 0.0};
    CU(cudaMemcpy(ctx->tc, init, sizeof(init), cudaMemcpyHostToDevice));
    return 0;
}

// ---- implicit incompressible SPH (iisph_kernels.cuh) -----------------------------------------
// A list consumer of the evaluation, like the EDAC and elastic-dynamics passes: it may run on a
// deferred drift check that the caller confirms afterwards (the evaluation is then repeated), so
// it does not wait for that check itself.  Everything it writes is overwritten by a repeat but
// the pressure, the warm start of the next solve: a repeat starts from p = p0 again.
int b200sph_iisph_pass(b200sph_ctx *ctx, const b200sph_iisph_program *prog, int64_t *pairs_out)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    const unsigned fm = prog->fluid_mask, sm = prog->solid_mask;
    if (fm == 0 || fm >= (1u << ctx->narr)) return set_err(ctx, "iisph_pass: bad fluid mask 0x%x", fm);
    if (sm >= (1u << ctx->narr) || (sm & fm)) return set_err(ctx, "iisph_pass: bad solid mask 0x%x (fluids 0x%x)", sm, fm);
    if (prog->min_iterations < 0 || prog->max_iterations < 1)
        return set_err(ctx, "iisph_pass: iterations must be min >= 0, max >= 1 (got %d, %d)", prog->min_iterations, prog->max_iterations);
    if (ctx->dim < 2) return set_err(ctx, "iisph_pass: IISPH runs in 2-D and 3-D");
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "iisph_pass runs on one GPU (no slab decomposition)");
    if (mirror_any(ctx)) return set_err(ctx, "iisph_pass: mirror domains are not supported");
    for (int a = 0; a < ctx->narr; a++)
        if (ctx->arr[a].n != ctx->arr[a].n_real)
            return set_err(ctx, "iisph_pass: array '%s' has ghost particles (the pressure iterations do not refresh them)", ctx->arr[a].name.c_str());
    if (!ctx->grid_valid) return set_err(ctx, "iisph_pass: the NNPS is stale (particles were pushed, resized or moved); call nnps_update first");
    if ((rc = ensure_prop(ctx, B200SPH_UADV))) return rc;
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    if (prog->dt_device && (rc = ensure_tc(ctx))) return rc;
    if ((rc = grow(ctx, ctx->iisph_st, 1, 1))) return rc;
    if (ctx->iisph_restore) {
        // the first attempt of this evaluation solved p from p0: start again from there
        for (int a = 0; a < ctx->narr; a++)
            if (((fm >> a) & 1u) && ctx->arr[a].n > 0)
                CU(cudaMemcpyAsync(f64_ptr(ctx, B200SPH_PF) + ctx->arr[a].off, f64_ptr(ctx, B200SPH_PF0) + ctx->arr[a].off,
                                   8 * (size_t)ctx->arr[a].n, cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->iisph_restore = false;
    }
    ctx->iisph_spec = ctx->check_pending;
    CU(cudaMemsetAsync(ctx->iisph_st, 0, sizeof(IisphState), ctx->stream));
    if (ctx->n_sorted == 0) {
        if (pairs_out) *pairs_out = 0;
        return 0;
    }
    unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
    for (int a = 0; a < ctx->narr; a++) {
        if ((fm >> a) & 1u)
            for (int b = 0; b < ctx->narr; b++)
                if (((fm | sm) >> b) & 1u) want[a] |= 0xFFull << (8 * b);
        if ((sm >> a) & 1u) want[a] |= 0xFFull << (8 * a);
    }
    if ((rc = prepare_lists(ctx, want, "iisph_pass: the neighbour lists cannot index the particles"))) return rc;
    const size_t n = (size_t)ctx->n_sorted, np = (size_t)ctx->pool_end;
    int64_t nmax = 1;
    for (int a = 0; a < ctx->narr; a++) nmax = std::max<int64_t>(nmax, ctx->arr[a].n);
    const size_t nbr = (size_t)cdiv(nmax, IISPH_RED);
    if ((rc = grow(ctx, ctx->iisph_P, n, n)) || (rc = grow(ctx, ctx->iisph_pnext, np, np)) ||
        (rc = grow(ctx, ctx->iisph_part, 2 * nbr, 2 * nbr)))
        return rc;
    IisphArgs ia;
    memset(&ia, 0, sizeof(ia));
    ia.P = ctx->iisph_P;
    ia.perm = ctx->perm; ia.cnt = ctx->cnt; ia.lst = ctx->lst; ia.skey = ctx->skey; ia.stype = ctx->stype;
    ia.x = f64_ptr(ctx, B200SPH_X); ia.y = f64_ptr(ctx, B200SPH_Y); ia.z = f64_ptr(ctx, B200SPH_Z);
    ia.h = f64_ptr(ctx, B200SPH_H); ia.m = f64_ptr(ctx, B200SPH_M);
    ia.rho = f64_ptr(ctx, B200SPH_RHO); ia.rho_c = ia.rho;
    ia.u = f64_ptr(ctx, B200SPH_U); ia.v = f64_ptr(ctx, B200SPH_V); ia.w = f64_ptr(ctx, B200SPH_W);
    ia.V = f64_ptr(ctx, B200SPH_IISPH_V);
    ia.uadv = f64_ptr(ctx, B200SPH_UADV); ia.vadv = f64_ptr(ctx, B200SPH_VADV); ia.wadv = f64_ptr(ctx, B200SPH_WADV);
    ia.rho_adv = f64_ptr(ctx, B200SPH_RHO_ADV);
    ia.dii0 = f64_ptr(ctx, B200SPH_DII0); ia.dii1 = f64_ptr(ctx, B200SPH_DII1); ia.dii2 = f64_ptr(ctx, B200SPH_DII2);
    ia.aii = f64_ptr(ctx, B200SPH_AII);
    ia.dijpj0 = f64_ptr(ctx, B200SPH_DIJPJ0); ia.dijpj1 = f64_ptr(ctx, B200SPH_DIJPJ1); ia.dijpj2 = f64_ptr(ctx, B200SPH_DIJPJ2);
    ia.p = f64_ptr(ctx, B200SPH_PF); ia.p0 = f64_ptr(ctx, B200SPH_PF0);
    ia.piter = f64_ptr(ctx, B200SPH_PITER); ia.pnext = ctx->iisph_pnext; ia.comp = f64_ptr(ctx, B200SPH_COMPRESSION);
    ia.au = f32_ptr(ctx, B200SPH_AU); ia.av = f32_ptr(ctx, B200SPH_AV); ia.aw = f32_ptr(ctx, B200SPH_AW);
    ia.dt_cfl = f32_ptr(ctx, B200SPH_DT_CFL); ia.dt_force = f32_ptr(ctx, B200SPH_DT_FORCE);
    ia.st = ctx->iisph_st; ia.part = ctx->iisph_part;
    ia.n = ctx->n_sorted; ia.capg = ctx->capg;
    ia.ncx = ctx->G.nc[0]; ia.ncy = ctx->G.nc[1]; ia.zorder = ctx->G.zorder;
    for (int d = 0; d < 3; d++) {
        ia.per[d] = ctx->G.periodic[d];
        ia.L[d] = ctx->dom_hi[d] - ctx->dom_lo[d];
    }
    ia.kr = ctx->radius_scale;
    ia.kfac = kernel_fac(ctx->kernel, ctx->dim);
    ia.fluid_mask = fm; ia.solid_mask = sm;
    ia.rho0 = prog->rho0; ia.nu = prog->nu; ia.gx = prog->gx; ia.gy = prog->gy; ia.gz = prog->gz;
    ia.omega = prog->omega; ia.tol = prog->tolerance;
    ia.min_it = prog->min_iterations; ia.max_it = prog->max_iterations;
    ia.dt = prog->dt; ia.tc = prog->dt_device ? ctx->tc : nullptr;
    if ((rc = pairs_arm(ctx, pairs_out, &ia.pair_counter))) return rc;
    PhaseTimer pt(ctx, 2);
    k_iisph_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(ia);
    LAUNCH_CHECK();
    const unsigned nb = (unsigned)cdiv(ctx->n_sorted, IISPH_NT);
    const auto pass = [&](const int which) {
        return with_kernel_dim(ctx, "iisph_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            switch (which) {
            case IISPH_V: k_iisph<K, D, IISPH_V><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            case IISPH_RHO: k_iisph<K, D, IISPH_RHO><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            case IISPH_ADV: k_iisph<K, D, IISPH_ADV><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            case IISPH_AII: k_iisph<K, D, IISPH_AII><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            case IISPH_DIJPJ: k_iisph<K, D, IISPH_DIJPJ><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            case IISPH_SOLVE: k_iisph<K, D, IISPH_SOLVE><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            default: k_iisph<K, D, IISPH_FORCE><<<nb, IISPH_NT, 0, ctx->stream>>>(ia); break;
            }
            LAUNCH_CHECK();
            return 0;
        });
    };
    if (sm && (rc = pass(IISPH_V))) return rc;
    if ((rc = pass(IISPH_RHO)) || (rc = pass(IISPH_ADV)) || (rc = pass(IISPH_AII))) return rc;
    int last = 0;
    for (int a = 0; a < ctx->narr; a++)
        if ((fm >> a) & 1u) last = a;
    pt.to(1);
    for (int it = 0; it < prog->max_iterations; it++) {
        if ((rc = pass(IISPH_DIJPJ))) return rc;
        for (int a = 0; a < ctx->narr; a++) {
            if (!((fm >> a) & 1u)) continue;
            ia.dest_mask = 1u << a;
            if ((rc = pass(IISPH_SOLVE))) return rc;
            if (ctx->arr[a].n > 0) {
                k_iisph_commit<<<(unsigned)cdiv(ctx->arr[a].n, 256), 256, 0, ctx->stream>>>(ia, ctx->arr[a].off, ctx->arr[a].n);
                LAUNCH_CHECK();
            }
        }
        for (int a = 0; a < ctx->narr; a++) {
            if (!((fm >> a) & 1u)) continue;
            const long long nba = std::max<long long>(1, cdiv(ctx->arr[a].n, IISPH_RED));
            if (ctx->arr[a].n > 0) {
                k_iisph_partials<<<(unsigned)nba, IISPH_RED, 0, ctx->stream>>>(ia, ctx->arr[a].off, ctx->arr[a].n);
                LAUNCH_CHECK();
            }
            k_iisph_converge<<<1, IISPH_RED, 0, ctx->stream>>>(ia, ctx->arr[a].n > 0 ? nba : 0, a, a == last);
            LAUNCH_CHECK();
        }
        ctx->stats.pair_launches++;
    }
    if ((rc = pass(IISPH_FORCE))) return rc;
    pt.stop();
    // rho, p and the accelerations changed: the next evaluation packs its records from the pool
    state_changed(ctx);
    ctx->spec_records = false;
    return pairs_read(ctx, pairs_out);
}

int b200sph_iisph_stats(b200sph_ctx *ctx, int *iterations, double compression[B200SPH_MAX_ARRAYS])
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->iisph_st) return set_err(ctx, "iisph_stats: no IISPH evaluation has run");
    IisphState st;
    CU(cudaMemcpyAsync(&st, ctx->iisph_st, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    *iterations = st.it;
    for (int a = 0; a < B200SPH_MAX_ARRAYS; a++) compression[a] = st.comp[a];
    return 0;
}

static int stage_iisph_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt)
{
    int rc = stage_begin(ctx, "stage_iisph", arr, which, devdt);
    if (rc) return rc;
    if (which != 1) return set_err(ctx, "stage_iisph: IISPHStep has stage1 only (which = 1, got %d)", which);
    if ((rc = ensure_prop(ctx, B200SPH_UADV))) return rc;
    PhaseTimer pt(ctx, 2);
    StageIisphArgs sa;
    sa.x = f64_ptr(ctx, B200SPH_X); sa.y = f64_ptr(ctx, B200SPH_Y); sa.z = f64_ptr(ctx, B200SPH_Z);
    sa.u = f64_ptr(ctx, B200SPH_U); sa.v = f64_ptr(ctx, B200SPH_V); sa.w = f64_ptr(ctx, B200SPH_W);
    sa.uadv = f64_ptr(ctx, B200SPH_UADV); sa.vadv = f64_ptr(ctx, B200SPH_VADV); sa.wadv = f64_ptr(ctx, B200SPH_WADV);
    sa.au = f32_ptr(ctx, B200SPH_AU); sa.av = f32_ptr(ctx, B200SPH_AV); sa.aw = f32_ptr(ctx, B200SPH_AW);
    sa.ptype = ctx->ptype;
    sa.pool_end = ctx->pool_end;
    sa.mask = arr < 0 ? ~0u : 1u << arr;
    sa.dt = dt;
    sa.tc = devdt ? ctx->tc : nullptr;
    if (ctx->pool_end > 0) {
        k_stage_iisph<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    particles_moved(ctx);
    return 0;
}
int b200sph_stage_iisph(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_iisph_impl(ctx, arr, which, dt, false); }
int b200sph_stage_iisph_dev(b200sph_ctx *ctx, int arr, int which) { return stage_iisph_impl(ctx, arr, which, 0.0, true); }

// ---- the generalised transport-velocity formulation (gtvf_kernels.cuh) -------------------------
// A list consumer like the IISPH pass.  Evaluation 0 runs without a neighbour-search update
// (GTVFIntegrator, gtvf.py:57): the positions are those of the last update, so the lists of that
// update serve it as they are.  Evaluation 1 may run on a deferred drift check; CorrectDensity
// moves rho into rho0 before it rewrites rho, so a repeat after a failed check keeps rho0 (the
// density stage 2 produced) instead of taking the first attempt's rho.
int b200sph_gtvf_pass(b200sph_ctx *ctx, const b200sph_gtvf_program *prog, int evaluation)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    const unsigned fm = prog->fluid_mask, sm = prog->solid_mask;
    if (evaluation != 0 && evaluation != 1) return set_err(ctx, "gtvf_pass: evaluation must be 0 or 1 (got %d)", evaluation);
    if (fm == 0 || fm >= (1u << ctx->narr) || (fm & (fm - 1)))
        return set_err(ctx, "gtvf_pass: bad fluid mask 0x%x (one fluid array)", fm);
    if (sm >= (1u << ctx->narr) || (sm & fm)) return set_err(ctx, "gtvf_pass: bad solid mask 0x%x (fluid 0x%x)", sm, fm);
    if (prog->nu > 0.0 && sm) return set_err(ctx, "gtvf_pass: nu > 0 with walls (SolidWallNoSlipBC reads a V the fluid does not have)");
    if (!(prog->pref != 0.0) || !(prog->rho0 != 0.0)) return set_err(ctx, "gtvf_pass: pref and rho0 must be non-zero");
    if (ctx->dim < 2) return set_err(ctx, "gtvf_pass: GTVF runs in 2-D and 3-D");
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "gtvf_pass runs on one GPU (no slab decomposition)");
    if (mirror_any(ctx)) return set_err(ctx, "gtvf_pass: mirror domains are not supported");
    for (int a = 0; a < ctx->narr; a++)
        if (ctx->arr[a].n != ctx->arr[a].n_real)
            return set_err(ctx, "gtvf_pass: array '%s' has ghost particles", ctx->arr[a].name.c_str());
    if (!ctx->grid_valid) return set_err(ctx, "gtvf_pass: the NNPS is stale (particles were pushed, resized or moved); call nnps_update first");
    if ((rc = ensure_prop(ctx, B200SPH_RHODIV))) return rc;
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    if (evaluation == 1) {
        // CorrectDensity.initialize (gtvf.py:138-141): rho0 = rho -- unless this is the repeat of
        // an evaluation whose drift check failed, which already did it
        if (!ctx->gtvf_restore)
            for (int a = 0; a < ctx->narr; a++)
                if (((fm >> a) & 1u) && ctx->arr[a].n > 0)
                    CU(cudaMemcpyAsync(f64_ptr(ctx, B200SPH_RHO0) + ctx->arr[a].off, f64_ptr(ctx, B200SPH_RHO) + ctx->arr[a].off,
                                       8 * (size_t)ctx->arr[a].n, cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->gtvf_restore = false;
        ctx->gtvf_spec = ctx->check_pending;
    }
    if (ctx->n_sorted == 0) return 0;
    unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
    for (int a = 0; a < ctx->narr; a++) {
        if ((fm >> a) & 1u)
            for (int b = 0; b < ctx->narr; b++)
                if (((fm | sm) >> b) & 1u) want[a] |= 0xFFull << (8 * b);
        if ((sm >> a) & 1u)
            for (int b = 0; b < ctx->narr; b++)
                if (((fm | sm) >> b) & 1u) want[a] |= 0xFFull << (8 * b);
    }
    if ((rc = prepare_lists(ctx, want, "gtvf_pass: the neighbour lists cannot index the particles"))) return rc;
    const size_t n = (size_t)ctx->n_sorted;
    if ((rc = grow(ctx, ctx->gtvf_P, n, n))) return rc;
    GtvfArgs ga;
    memset(&ga, 0, sizeof(ga));
    ga.P = ctx->gtvf_P;
    ga.perm = ctx->perm; ga.cnt = ctx->cnt; ga.lst = ctx->lst; ga.skey = ctx->skey; ga.stype = ctx->stype;
    ga.x = f64_ptr(ctx, B200SPH_X); ga.y = f64_ptr(ctx, B200SPH_Y); ga.z = f64_ptr(ctx, B200SPH_Z);
    ga.h = f64_ptr(ctx, B200SPH_H); ga.m = f64_ptr(ctx, B200SPH_M);
    ga.u = f64_ptr(ctx, B200SPH_U); ga.v = f64_ptr(ctx, B200SPH_V); ga.w = f64_ptr(ctx, B200SPH_W);
    // a fluid's uhat .. what and a wall's ug .. wg share the transport-velocity slots
    ga.uh = f64_ptr(ctx, B200SPH_UHAT); ga.vh = f64_ptr(ctx, B200SPH_VHAT); ga.wh = f64_ptr(ctx, B200SPH_WHAT);
    ga.ug = f64_ptr(ctx, B200SPH_UHAT); ga.vg = f64_ptr(ctx, B200SPH_VHAT); ga.wg = f64_ptr(ctx, B200SPH_WHAT);
    ga.rho = f64_ptr(ctx, B200SPH_RHO); ga.rho0 = f64_ptr(ctx, B200SPH_RHO0);
    ga.pf = f64_ptr(ctx, B200SPH_PF); ga.rhodiv = f64_ptr(ctx, B200SPH_RHODIV); ga.p0 = f64_ptr(ctx, B200SPH_GTVF_P0);
    ga.p = f32_ptr(ctx, B200SPH_P); ga.arho = f32_ptr(ctx, B200SPH_ARHO);
    ga.au = f32_ptr(ctx, B200SPH_AU); ga.av = f32_ptr(ctx, B200SPH_AV); ga.aw = f32_ptr(ctx, B200SPH_AW);
    // a fluid's auhat .. awhat and a wall's uf .. wf share these slots too
    ga.auh = f32_ptr(ctx, B200SPH_AUHAT); ga.avh = f32_ptr(ctx, B200SPH_AVHAT); ga.awh = f32_ptr(ctx, B200SPH_AWHAT);
    ga.uf = f32_ptr(ctx, B200SPH_AUHAT); ga.vf = f32_ptr(ctx, B200SPH_AVHAT); ga.wf = f32_ptr(ctx, B200SPH_AWHAT);
    ga.vol = f32_ptr(ctx, B200SPH_VOL); ga.wij = f32_ptr(ctx, B200SPH_PAVG);
    ga.n = ctx->n_sorted; ga.capg = ctx->capg;
    ga.ncx = ctx->G.nc[0]; ga.ncy = ctx->G.nc[1]; ga.zorder = ctx->G.zorder;
    for (int d = 0; d < 3; d++) {
        ga.per[d] = ctx->G.periodic[d];
        ga.L[d] = ctx->dom_hi[d] - ctx->dom_lo[d];
    }
    ga.kr = ctx->radius_scale;
    ga.kfac = kernel_fac(ctx->kernel, ctx->dim);
    ga.fluid_mask = fm; ga.solid_mask = sm;
    ga.rho0c = prog->rho0; ga.pref = prog->pref; ga.c0 = prog->c0; ga.alpha = prog->alpha; ga.nu = prog->nu;
    ga.gx = prog->gx; ga.gy = prog->gy; ga.gz = prog->gz;
    PhaseTimer pt(ctx, 2);
    k_gtvf_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(ga);
    LAUNCH_CHECK();
    const unsigned nb = (unsigned)cdiv(ctx->n_sorted, GTVF_NT);
    const auto pass = [&](const int which) {
        return with_kernel_dim(ctx, "gtvf_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            switch (which) {
            case GTVF_WALLV: k_gtvf<K, D, GTVF_WALLV><<<nb, GTVF_NT, 0, ctx->stream>>>(ga); break;
            case GTVF_CONT: k_gtvf<K, D, GTVF_CONT><<<nb, GTVF_NT, 0, ctx->stream>>>(ga); break;
            case GTVF_RHO: k_gtvf<K, D, GTVF_RHO><<<nb, GTVF_NT, 0, ctx->stream>>>(ga); break;
            case GTVF_WALLP: k_gtvf<K, D, GTVF_WALLP><<<nb, GTVF_NT, 0, ctx->stream>>>(ga); break;
            default: k_gtvf<K, D, GTVF_MOM><<<nb, GTVF_NT, 0, ctx->stream>>>(ga); break;
            }
            LAUNCH_CHECK();
            return 0;
        });
    };
    if (evaluation == 0) {
        if (sm && (rc = pass(GTVF_WALLV))) return rc;
        if ((rc = pass(GTVF_CONT))) return rc;
    } else {
        if ((rc = pass(GTVF_RHO))) return rc;
        if (sm && (rc = pass(GTVF_WALLP))) return rc;
        if ((rc = pass(GTVF_MOM))) return rc;
    }
    ctx->stats.pair_launches++;
    pt.stop();
    // rho, p and the accelerations changed: the next evaluation packs its records from the pool
    state_changed(ctx);
    ctx->spec_records = false;
    return 0;
}

static int stage_gtvf_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt)
{
    int rc = stage_begin(ctx, "stage_gtvf", arr, which, devdt, 3);
    if (rc) return rc;
    if (which < 1) return set_err(ctx, "stage_gtvf: GTVFStep has stages 1, 2 and 3 (got %d)", which);
    PhaseTimer pt(ctx, 2);
    StageGtvfArgs sa;
    sa.x = f64_ptr(ctx, B200SPH_X); sa.y = f64_ptr(ctx, B200SPH_Y); sa.z = f64_ptr(ctx, B200SPH_Z);
    sa.u = f64_ptr(ctx, B200SPH_U); sa.v = f64_ptr(ctx, B200SPH_V); sa.w = f64_ptr(ctx, B200SPH_W);
    sa.uh = f64_ptr(ctx, B200SPH_UHAT); sa.vh = f64_ptr(ctx, B200SPH_VHAT); sa.wh = f64_ptr(ctx, B200SPH_WHAT);
    sa.rho = f64_ptr(ctx, B200SPH_RHO);
    sa.au = f32_ptr(ctx, B200SPH_AU); sa.av = f32_ptr(ctx, B200SPH_AV); sa.aw = f32_ptr(ctx, B200SPH_AW);
    sa.auh = f32_ptr(ctx, B200SPH_AUHAT); sa.avh = f32_ptr(ctx, B200SPH_AVHAT); sa.awh = f32_ptr(ctx, B200SPH_AWHAT);
    sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    sa.ptype = ctx->ptype;
    sa.pool_end = ctx->pool_end;
    sa.mask = arr < 0 ? ~0u : 1u << arr;
    sa.which = which;
    sa.dt = dt;
    sa.tc = devdt ? ctx->tc : nullptr;
    if (ctx->pool_end > 0) {
        k_stage_gtvf<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    // stages 1 and 3 change velocities only: the lists stay valid for evaluation 0, which runs
    // without a neighbour-search update
    if (which == 2) particles_moved(ctx);
    else state_changed(ctx);
    return 0;
}
int b200sph_stage_gtvf(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_gtvf_impl(ctx, arr, which, dt, false); }
int b200sph_stage_gtvf_dev(b200sph_ctx *ctx, int arr, int which) { return stage_gtvf_impl(ctx, arr, which, 0.0, true); }

// ---- conservative reproducing-kernel SPH (crksph_kernels.cuh) ----------------------------------
// A list consumer like the GTVF pass.  Evaluation 0 runs on a deferred drift check after stage 3
// moved the particles; everything it reads besides positions, velocities and e is written by an
// earlier pass of the same evaluation (the first StateEquation's p and cs are overwritten before
// anything reads them), so a repeat after a failed check needs nothing restored.  Evaluation 1
// follows stage 2, which moves no particle, and writes ae only.
int b200sph_crksph_pass(b200sph_ctx *ctx, const b200sph_crksph_program *prog, int evaluation)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    const unsigned fm = prog->fluid_mask;
    if (evaluation != 0 && evaluation != 1) return set_err(ctx, "crksph_pass: evaluation must be 0 or 1 (got %d)", evaluation);
    if (fm == 0 || fm >= (1u << ctx->narr) || (fm & (fm - 1)))
        return set_err(ctx, "crksph_pass: bad fluid mask 0x%x (one fluid array)", fm);
    if (ctx->dim < 2) return set_err(ctx, "crksph_pass: CRKSPH runs in 2-D and 3-D");
    if (ctx->peer_box || ctx->comm_pending) return set_err(ctx, "crksph_pass runs on one GPU (no slab decomposition)");
    if (mirror_any(ctx)) return set_err(ctx, "crksph_pass: mirror domains are not supported");
    for (int a = 0; a < ctx->narr; a++)
        if (ctx->arr[a].n != ctx->arr[a].n_real)
            return set_err(ctx, "crksph_pass: array '%s' has ghost particles", ctx->arr[a].name.c_str());
    if (!ctx->grid_valid) return set_err(ctx, "crksph_pass: the NNPS is stale (particles were pushed, resized or moved); call nnps_update first");
    if ((rc = ensure_prop(ctx, B200SPH_CRK_E))) return rc;
    if ((rc = eos_flush(ctx)) || (rc = ab_positions(ctx))) return rc;
    if (ctx->n_sorted == 0) return 0;
    unsigned long long want[B200SPH_MAX_ARRAYS] = {0};
    for (int a = 0; a < ctx->narr; a++)
        if ((fm >> a) & 1u) want[a] = 0xFFull << (8 * a);
    if ((rc = prepare_lists(ctx, want, "crksph_pass: the neighbour lists cannot index the particles"))) return rc;
    const size_t n = (size_t)ctx->n_sorted;
    if ((rc = grow(ctx, ctx->crk_P, n, n))) return rc;
    CrkArgs ca;
    memset(&ca, 0, sizeof(ca));
    ca.P = ctx->crk_P;
    ca.perm = ctx->perm; ca.cnt = ctx->cnt; ca.lst = ctx->lst; ca.skey = ctx->skey; ca.stype = ctx->stype;
    ca.h = f64_ptr(ctx, B200SPH_H); ca.m = f64_ptr(ctx, B200SPH_M);
    ca.u = f64_ptr(ctx, B200SPH_U); ca.v = f64_ptr(ctx, B200SPH_V); ca.w = f64_ptr(ctx, B200SPH_W);
    ca.u0 = f64_ptr(ctx, B200SPH_U0); ca.v0 = f64_ptr(ctx, B200SPH_V0); ca.w0 = f64_ptr(ctx, B200SPH_W0);
    ca.rho = f64_ptr(ctx, B200SPH_RHO); ca.p = f64_ptr(ctx, B200SPH_PF);
    ca.e = f64_ptr(ctx, B200SPH_CRK_E); ca.ae = f64_ptr(ctx, B200SPH_CRK_AE); ca.cs = f64_ptr(ctx, B200SPH_CRK_CS);
    ca.V = f64_ptr(ctx, B200SPH_CRK_V); ca.ai = f64_ptr(ctx, B200SPH_CRK_AI);
    ca.au = f64_ptr(ctx, B200SPH_CRK_AU); ca.av = f64_ptr(ctx, B200SPH_CRK_AV); ca.aw = f64_ptr(ctx, B200SPH_CRK_AW);
    for (int k = 0; k < 3; k++) {
        ca.bi[k] = f64_ptr(ctx, B200SPH_CRK_BI0 + k);
        ca.gai[k] = f64_ptr(ctx, B200SPH_CRK_GRADAI0 + k);
    }
    for (int k = 0; k < 9; k++) {
        ca.gbi[k] = f64_ptr(ctx, B200SPH_CRK_GRADBI00 + k);
        ca.gv[k] = f64_ptr(ctx, B200SPH_CRK_GRADV00 + k);
    }
    ca.n = ctx->n_sorted; ca.capg = ctx->capg;
    ca.ncx = ctx->G.nc[0]; ca.ncy = ctx->G.nc[1]; ca.zorder = ctx->G.zorder;
    for (int d = 0; d < 3; d++) {
        ca.per[d] = ctx->G.periodic[d];
        ca.L[d] = ctx->dom_hi[d] - ctx->dom_lo[d];
    }
    ca.kr = ctx->radius_scale;
    ca.kfac = kernel_fac(ctx->kernel, ctx->dim);
    ca.fluid_mask = fm;
    ca.gamma = prog->gamma; ca.gx = prog->gx; ca.gy = prog->gy; ca.gz = prog->gz;
    ca.cl = prog->cl; ca.cq = prog->cq; ca.eta_crit = prog->eta_crit; ca.eta_fold = prog->eta_fold;
    ca.cl_e = prog->cl_e; ca.cq_e = prog->cq_e; ca.eta_crit_e = prog->eta_crit_e; ca.eta_fold_e = prog->eta_fold_e;
    ca.nu = prog->nu; ca.eta = prog->eta;
    PhaseTimer pt(ctx, 2);
    k_crksph_pack<<<(unsigned)cdiv(ctx->n_sorted, 256), 256, 0, ctx->stream>>>(
        ca, f64_ptr(ctx, B200SPH_X), f64_ptr(ctx, B200SPH_Y), f64_ptr(ctx, B200SPH_Z));
    LAUNCH_CHECK();
    const unsigned nb = (unsigned)cdiv(ctx->n_sorted, CRK_NT);
    const auto pass = [&](const int which) {
        return with_kernel_dim(ctx, "crksph_pass", [&](auto kc, auto dc) {
            constexpr int K = decltype(kc)::value, D = decltype(dc)::value;
            if constexpr (D >= 2) {
                switch (which) {
                case CRK_VOL: k_crksph<K, D, CRK_VOL><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                case CRK_PRE: k_crksph<K, D, CRK_PRE><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                case CRK_RHO: k_crksph<K, D, CRK_RHO><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                case CRK_GRADV: k_crksph<K, D, CRK_GRADV><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                case CRK_MOM: k_crksph<K, D, CRK_MOM><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                default: k_crksph<K, D, CRK_ENERGY><<<nb, CRK_NT, 0, ctx->stream>>>(ca); break;
                }
                LAUNCH_CHECK();
            }
            return 0;
        });
    };
    if (evaluation == 0) {
        for (const int which : {CRK_VOL, CRK_PRE, CRK_RHO, CRK_GRADV, CRK_MOM})
            if ((rc = pass(which))) return rc;
    } else if ((rc = pass(CRK_ENERGY))) {
        return rc;
    }
    ctx->stats.pair_launches++;
    pt.stop();
    state_changed(ctx);
    ctx->spec_records = false;
    return 0;
}

static int stage_crksph_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt)
{
    int rc = stage_begin(ctx, "stage_crksph", arr, which, devdt, 3);
    if (rc) return rc;
    if (which < 1) return set_err(ctx, "stage_crksph: CRKSPHStep has stages 1, 2 and 3 (got %d)", which);
    if ((rc = ensure_prop(ctx, B200SPH_CRK_E))) return rc;
    PhaseTimer pt(ctx, 2);
    StageCrkArgs sa;
    sa.x = f64_ptr(ctx, B200SPH_X); sa.y = f64_ptr(ctx, B200SPH_Y); sa.z = f64_ptr(ctx, B200SPH_Z);
    sa.u = f64_ptr(ctx, B200SPH_U); sa.v = f64_ptr(ctx, B200SPH_V); sa.w = f64_ptr(ctx, B200SPH_W);
    sa.u0 = f64_ptr(ctx, B200SPH_U0); sa.v0 = f64_ptr(ctx, B200SPH_V0); sa.w0 = f64_ptr(ctx, B200SPH_W0);
    sa.e = f64_ptr(ctx, B200SPH_CRK_E); sa.ae = f64_ptr(ctx, B200SPH_CRK_AE);
    sa.au = f64_ptr(ctx, B200SPH_CRK_AU); sa.av = f64_ptr(ctx, B200SPH_CRK_AV); sa.aw = f64_ptr(ctx, B200SPH_CRK_AW);
    sa.ptype = ctx->ptype;
    sa.pool_end = ctx->pool_end;
    sa.mask = arr < 0 ? ~0u : 1u << arr;
    sa.which = which;
    sa.dt = dt;
    sa.tc = devdt ? ctx->tc : nullptr;
    if (ctx->pool_end > 0) {
        k_stage_crksph<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    // only stage 3 moves particles: after stages 1 and 2 the lists stay valid for the evaluation
    // that follows
    if (which == 3) particles_moved(ctx);
    else state_changed(ctx);
    return 0;
}
int b200sph_stage_crksph(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_crksph_impl(ctx, arr, which, dt, false); }
int b200sph_stage_crksph_dev(b200sph_ctx *ctx, int arr, int which) { return stage_crksph_impl(ctx, arr, which, 0.0, true); }

// the fused stage kernel applies when one launch steps every array (arr == -1) and the
// neighbour lists of the current build can be reused: then the records of the next
// evaluation can be written at the particles' frozen sorted slots
static bool can_fuse_stage(const b200sph_ctx *ctx, int arr)
{
    if (!ctx->fuse || arr != -1 || !reusable_build(ctx) || ctx->n_sorted <= 0) return false;
    if (ctx->periodic[0] || ctx->periodic[1] || ctx->periodic[2] || mirror_any(ctx)) return false;
    int64_t ntot = 0;
    for (int a = 0; a < ctx->narr; a++) ntot += ctx->arr[a].n;
    return ntot == ctx->n_sorted && lists_usable(ctx, ntot);
}

// WCSPHStep (rk3 = false: stages 1, 2) and WCSPHTVDRK3Step (rk3: stages 1, 2, 3); the dt
// factors belong to the evaluation before the stepper's last stage
static int stage_impl(b200sph_ctx *ctx, int arr, int which, double dt, bool devdt, bool rk3 = false)
{
    const int last = rk3 ? 3 : 2;
    int rc = stage_begin(ctx, rk3 ? "stage_rk3" : "stage", arr, which, devdt, last, true);
    if (rc) return rc;
    const bool fused = ctx->pool_end > 0 && can_fuse_stage(ctx, arr);
    // a pending half step: only the fused stage 2 that follows it, with the same kind of dt, reads
    // neither x .. w nor p / cs, and forms the predicted rho itself
    const bool takes_half = ctx->half_pending && fused && which == 2 && !rk3 && ctx->rec32 &&
                            (devdt ? ctx->tc : nullptr) == ctx->half_tc;
    if (!takes_half && (rc = half_materialise(ctx))) return rc;
    // EOS calls issued since the last pair pass, or any before an initialize (which copies the
    // rho they clamp), go to the pool now; the pool side a pair pass left is the fused kernel's
    if ((which == 0 || !fused || ctx->eos_any) && (rc = eos_flush(ctx))) return rc;
    if (which == 0 && fused && !ctx->peer_box) {   // waits for the fused stage (init_materialise)
        ctx->init_pending = true;
        return 0;
    }
    PhaseTimer pt(ctx, 2);
    int do_init = ctx->init_pending ? INIT_COPY : INIT_NONE;
    if (which != 0 && fused && ctx->init_pending && init_by_rename(ctx, which)) {
        for (int k = 0; k <= B200SPH_RHO - B200SPH_X; k++) std::swap(ctx->prop[B200SPH_X + k], ctx->prop[B200SPH_X0 + k]);
        do_init = INIT_RENAMED;
    }
    StageArgs sa;
    stage_args(ctx, sa, arr, which, dt, devdt);
    if (rk3) sa.f = dt;   // every TVD-RK3 stage takes the whole dt
    sa.rho = f64_ptr(ctx, B200SPH_RHO); sa.rho0 = f64_ptr(ctx, B200SPH_RHO0); sa.arho = f32_ptr(ctx, B200SPH_ARHO);
    if (which != 0 && fused) {
        // stage + records of the next evaluation (+ the dt factors after the last stage) in one pass
        FusePackArgs q;
        memset(&q, 0, sizeof(q));
        q.h = f64_ptr(ctx, B200SPH_H); q.m = f64_ptr(ctx, B200SPH_M);
        q.p = f32_ptr(ctx, B200SPH_P); q.cs = f32_ptr(ctx, B200SPH_CS);
        q.rank = ctx->rank; q.key_of = ctx->key_of;
        q.A0 = ctx->A0; q.AB = ctx->AB; q.C = ctx->C;
        q.R = ctx->rec32 ? ctx->R.p : nullptr;   // the layout the last pair pass read
        if (q.R && ctx->hm_known && !std::isnan(ctx->h_uniform)) {   // 8 B per particle less to read
            q.h = nullptr;
            q.h_uniform = ctx->h_uniform;
        }
        q.E32 = ctx->rec32_eos;
        q.G = ctx->G;
        q.red_u32 = ctx->red_u32;
        q.dt_cfl = f32_ptr(ctx, B200SPH_DT_CFL); q.dt_force = f32_ptr(ctx, B200SPH_DT_FORCE);
        q.red = ctx->red;
        q.do_init = do_init;
        q.reduce_dt = (which == last && ctx->dt_adaptive_seen) ? 1 : 0;
        q.eos_any = ctx->eos_last_valid ? 1 : 0;
        q.E = ctx->eos_last;
        q.eos_pool = ctx->eos_pool_any ? 1 : 0;
        q.EP = ctx->eos_pool;
        q.half_pending = (do_init == INIT_RENAMED && !rk3 && q.R) ? 1 : 0;
        if (takes_half && ctx->half_pending) {   // (still pending: eos_flush above may have formed it)
            q.arho_half = ctx->acc_swapped ? ctx->acc_spare[0].p : f32_ptr(ctx, B200SPH_ARHO);
            q.f_half = ctx->half_f;
        }
        ctx->half_pending = q.half_pending != 0;   // (stage 2 clears it)
        ctx->acc_swapped = false;
        if (ctx->half_pending) {
            ctx->half_f = sa.f, ctx->half_tc = sa.tc;
            ctx->half_eos = q.eos_pool, ctx->half_EP = q.EP;
        }
        ctx->init_pending = false;
        ctx->eos_pool_any = false;
        if (q.reduce_dt && !ctx->red_armed) {
            k_red_init<<<1, 32, 0, ctx->stream>>>(ctx->red);
            LAUNCH_CHECK();
        }
        CU(cudaMemsetAsync(ctx->red_u32, 0, 2 * sizeof(unsigned), ctx->stream));
        if (rk3) k_stage_pack_rk3<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa, q);
        else k_stage_pack<<<(unsigned)cdiv(ctx->pool_end, 256), 256, 0, ctx->stream>>>(sa, q);
        LAUNCH_CHECK();
        ctx->n_fused++;
        if (q.reduce_dt) ctx->red_armed = false;
        if (which == last) ctx->dt_reduced = q.reduce_dt != 0, ctx->dt_adaptive_seen = false;
        positions_changed(ctx);        // particles moved: nnps_update must decide about the lists
        ctx->packed_valid = true;      // ... but their packed positions are current,
        ctx->ab_stale = q.R != nullptr;    // (in R only, with the 32-byte records)
        ctx->drift_measured = true;    // the drift of the build is in red_u32,
        ctx->state_packed = true;      // and so is their packed state,
        ctx->spec_records = ctx->eos_last_valid;   // with last evaluation's EOS calls applied
        ctx->spec_confirmed = 0;
        return 0;
    }
    if ((rc = init_materialise(ctx))) return rc;
    if (ctx->pool_end > 0) {
        const unsigned nb = (unsigned)cdiv(ctx->pool_end, 256);
        if (rk3 && which != 0) k_stage_rk3<<<nb, 256, 0, ctx->stream>>>(sa);
        else k_stage<<<nb, 256, 0, ctx->stream>>>(sa);
        LAUNCH_CHECK();
    }
    if (which != 0) particles_moved(ctx);
    if (which == last) ctx->dt_adaptive_seen = false, ctx->dt_reduced = false;
    return 0;
}

int b200sph_stage(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_impl(ctx, arr, which, dt, false); }
int b200sph_stage_dev(b200sph_ctx *ctx, int arr, int which) { return stage_impl(ctx, arr, which, 0.0, true); }
int b200sph_stage_rk3(b200sph_ctx *ctx, int arr, int which, double dt) { return stage_impl(ctx, arr, which, dt, false, true); }
int b200sph_stage_rk3_dev(b200sph_ctx *ctx, int arr, int which) { return stage_impl(ctx, arr, which, 0.0, true, true); }

// ---- device-resident time step ------------------------------------------------
int b200sph_time_control(b200sph_ctx *ctx, double *external_block8, double **dev_block)
{
    CU(cudaSetDevice(ctx->device));
    if (int rc = half_materialise(ctx)) return rc;   // (its factor may be dt in this block)
    if (external_block8) {
        CU(ctx->tc_own.reset());
        ctx->tc = external_block8;
        const double init[8] = {0.0, 0.0, 1e20, -1.0, 0.0, 0.0, 0.0, 0.0};
        CU(cudaMemcpyAsync(ctx->tc, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    } else if (int rc = ensure_tc(ctx)) return rc;
    if (!ctx->tc_host) {
        if (int rc = grow(ctx, ctx->tc_host, 4, 4)) return rc;
        for (int i = 0; i < 2; i++) CU(cudaEventCreateWithFlags(&ctx->tc_evt[i], cudaEventDisableTiming));
    }
    if (dev_block) *dev_block = ctx->tc;
    return 0;
}

int b200sph_time_set(b200sph_ctx *ctx, double t, double dt)
{
    CU(cudaSetDevice(ctx->device));
    int rc = b200sph_time_control(ctx, nullptr, nullptr);
    if (rc) return rc;
    const double v[2] = {dt, t};
    CU(cudaMemcpyAsync(ctx->tc, v, sizeof(v), cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// max dt_cfl, max dt_force, min h into red[9,11,12] -- unless the fused stage2 kernel has
// just left them there
static int reduce_dt_factors(b200sph_ctx *ctx)
{
    if (ctx->dt_reduced) return 0;
    k_red_init<<<1, 32, 0, ctx->stream>>>(ctx->red);
    LAUNCH_CHECK();
    if (ctx->pool_end > 0) {
        const unsigned nb = (unsigned)std::min<int64_t>(cdiv(ctx->pool_end, 256), REDUCE_BLOCKS);
        k_reduce_dt<<<nb, 256, 0, ctx->stream>>>(f32_ptr(ctx, B200SPH_DT_CFL), f32_ptr(ctx, B200SPH_DT_FORCE), f64_ptr(ctx, B200SPH_H),
                                                 ctx->ptype, ctx->pool_end, ctx->red);
        LAUNCH_CHECK();
    }
    ctx->red_armed = false;
    return 0;
}

int b200sph_dt_propose(b200sph_ctx *ctx, double cfl, int fixed_h)
{
    if (int rcc = require_confirmed(ctx, "dt_propose")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, true, true);   // (dt_cfl, dt_force and h only)
    if (rc) return rc;
    if ((rc = b200sph_time_control(ctx, nullptr, nullptr))) return rc;
    PhaseTimer pt(ctx, 2);
    if ((rc = reduce_dt_factors(ctx))) return rc;
    k_dt_propose<<<1, 1, 0, ctx->stream>>>(ctx->red, ctx->tc, cfl, fixed_h);
    LAUNCH_CHECK();
    ctx->red_armed = true;
    ctx->dt_reduced = false;
    ctx->dt_adaptive_seen = true;
    return 0;
}

int b200sph_dt_advance(b200sph_ctx *ctx, double cfl, int fixed_h, double prev_factor, double new_factor, int adaptive, int advance,
                       int snapshot_slot)
{
    if (int rcc = require_confirmed(ctx, "dt_advance")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, true, true);   // (dt_cfl, dt_force and h only)
    if (rc) return rc;
    if ((rc = b200sph_time_control(ctx, nullptr, nullptr))) return rc;
    if (!(prev_factor > 0.0) || !(new_factor > 0.0)) return set_err(ctx, "dt_advance: damping factors must be positive");
    if (snapshot_slot > 1) return set_err(ctx, "dt_advance: snapshot slot must be 0 or 1");
    PhaseTimer pt(ctx, 2);
    if (adaptive && (rc = reduce_dt_factors(ctx))) return rc;
    k_dt_advance<<<1, 1, 0, ctx->stream>>>(ctx->red, ctx->tc, cfl, fixed_h, prev_factor, new_factor, adaptive, advance, ctx->t_final, ctx->t_eps);
    LAUNCH_CHECK();
    ctx->red_armed = true;
    ctx->dt_reduced = false;
    ctx->dt_adaptive_seen = adaptive != 0;
    if (snapshot_slot >= 0) {
        CU(cudaMemcpyAsync(ctx->tc_host + 2 * snapshot_slot, ctx->tc, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaEventRecord(ctx->tc_evt[snapshot_slot], ctx->stream));
    }
    return 0;
}

int b200sph_dt_commit(b200sph_ctx *ctx, double prev_factor, double new_factor, int in_parallel, int adaptive, int advance, int snapshot_slot)
{
    CU(cudaSetDevice(ctx->device));
    int rc = b200sph_time_control(ctx, nullptr, nullptr);
    if (rc) return rc;
    if (!(prev_factor > 0.0) || !(new_factor > 0.0)) return set_err(ctx, "dt_commit: damping factors must be positive");
    k_dt_commit<<<1, 1, 0, ctx->stream>>>(ctx->tc, prev_factor, new_factor, in_parallel, adaptive, advance, ctx->t_final, ctx->t_eps);
    LAUNCH_CHECK();
    if (snapshot_slot >= 0) {
        if (snapshot_slot > 1) return set_err(ctx, "dt_commit: snapshot slot must be 0 or 1");
        CU(cudaMemcpyAsync(ctx->tc_host + 2 * snapshot_slot, ctx->tc, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaEventRecord(ctx->tc_evt[snapshot_slot], ctx->stream));
    }
    return 0;
}

int b200sph_time_final(b200sph_ctx *ctx, double t_final, double eps)
{
    if (!(eps >= 0.0) || t_final != t_final) return set_err(ctx, "time_final: bad final time / tolerance");
    ctx->t_final = t_final;
    ctx->t_eps = eps;
    return 0;
}

int b200sph_time_snapshot(b200sph_ctx *ctx, int slot, double out[2])
{
    if (slot < 0 || slot > 1 || !ctx->tc_host) return set_err(ctx, "time_snapshot: no snapshot in slot %d", slot);
    CU(cudaSetDevice(ctx->device));
    CU(cudaEventSynchronize(ctx->tc_evt[slot]));
    out[0] = ctx->tc_host[2 * slot];      // dt of the step that follows the snapshot
    out[1] = ctx->tc_host[2 * slot + 1];  // t at the snapshot
    return 0;
}

int b200sph_time_get(b200sph_ctx *ctx, double out[2])
{
    CU(cudaSetDevice(ctx->device));
    int rc = b200sph_time_control(ctx, nullptr, nullptr);
    if (rc) return rc;
    double v[2];
    CU(cudaMemcpyAsync(v, ctx->tc, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    out[0] = v[0];
    out[1] = v[1];
    return 0;
}

int b200sph_dt_factors(b200sph_ctx *ctx, double out[3])
{
    if (int rcc = require_confirmed(ctx, "dt_factors")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx, true, true);   // (dt_cfl, dt_force and h only)
    if (rc) return rc;
    PhaseTimer pt(ctx, 2);
    if ((rc = reduce_dt_factors(ctx))) return rc;
    ctx->dt_adaptive_seen = true;
    CU(cudaMemcpyAsync(ctx->red_host, ctx->red, 16 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const double mc = o2d(ctx->red_host[9]), mf = o2d(ctx->red_host[11]), hm = o2d(ctx->red_host[12]);
    out[0] = mc < -1e299 ? -1.0 : mc;  // _my_max of an empty property is -1.0, integrator.py:55-59
    out[1] = mf < -1e299 ? -1.0 : mf;
    out[2] = std::min(1.0, hm);        // compute_h_minimum starts from 1.0, integrator.py:149
    return 0;
}

// ---- halo helpers ------------------------------------------------------------
// The ghost and the migration message by property id, field by field: the first halo_nf /
// migrate_nf of these (the elastic-dynamics fields travel only when that group is allocated).
// An fp32 or integer property travels as a double.
static const int halo_msg[B200SPH_HALO_FIELDS_SOLID] = {
    B200SPH_X, B200SPH_Y, B200SPH_Z, B200SPH_U, B200SPH_V, B200SPH_W, B200SPH_RHO, B200SPH_H, B200SPH_M,
    B200SPH_S00, B200SPH_S01, B200SPH_S02, B200SPH_S11, B200SPH_S12, B200SPH_S22, B200SPH_CS};
static const int migrate_msg[B200SPH_MIGRATE_FIELDS_SOLID] = {
    B200SPH_X, B200SPH_Y, B200SPH_Z, B200SPH_U, B200SPH_V, B200SPH_W, B200SPH_RHO, B200SPH_H, B200SPH_M,
    B200SPH_X0, B200SPH_Y0, B200SPH_Z0, B200SPH_U0, B200SPH_V0, B200SPH_W0, B200SPH_RHO0, B200SPH_GID,
    B200SPH_S00, B200SPH_S01, B200SPH_S02, B200SPH_S11, B200SPH_S12, B200SPH_S22,
    B200SPH_S000, B200SPH_S010, B200SPH_S020, B200SPH_S110, B200SPH_S120, B200SPH_S220, B200SPH_CS};

// the halo kernels' view of the ghost message: its fp64 fields, then cs
static HaloPtrs halo_ptrs(b200sph_ctx *ctx)
{
    HaloPtrs P;
    for (int f = 0; f < B200SPH_HALO_FIELDS_SOLID - 1; f++) P.p[f] = f64_ptr(ctx, halo_msg[f]);
    P.cs = f32_ptr(ctx, halo_msg[B200SPH_HALO_FIELDS_SOLID - 1]);
    return P;
}

// zero particles [o, o + n) of the allocated properties among ids first .. last
static int zero_props(b200sph_ctx *ctx, int first, int last, int64_t o, int64_t n)
{
    for (int p = first; p <= last; p++) {
        const size_t esz = prop_kind(p).size();
        if (ctx->prop[p]) CU(cudaMemsetAsync((char *)ctx->prop[p] + esz * (size_t)o, 0, esz * (size_t)n, ctx->stream));
    }
    return 0;
}

// What the particles [o, o + n) that arrive by a message get for the properties it does not carry:
// the derived fp32 fields (of the elastic-dynamics group too, when it is allocated) zero; with the
// ghost message (no stage copies, no gid) the stage copies zero and gid 0xFFFFFFFF; tag `tag`; pid 0.
// Called before the message is written: an elastic array's cs comes with it.
static int arrival_init(b200sph_ctx *ctx, int64_t o, int64_t n, bool ghost_msg, uint32_t tag)
{
    const unsigned nb = (unsigned)cdiv(n, 256);
    int rc;
    if ((rc = zero_props(ctx, B200SPH_P, B200SPH_DT_FORCE, o, n)) || (rc = zero_props(ctx, B200SPH_V00, B200SPH_AS22, o, n)))
        return rc;
    if (ghost_msg) {
        if ((rc = zero_props(ctx, B200SPH_X0, B200SPH_RHO0, o, n)) || (rc = zero_props(ctx, B200SPH_S000, B200SPH_S220, o, n)))
            return rc;
        k_fill_u32<<<nb, 256, 0, ctx->stream>>>(u32_ptr(ctx, B200SPH_GID) + o, n, 0xFFFFFFFFu);
        LAUNCH_CHECK();
    }
    k_fill_u32<<<nb, 256, 0, ctx->stream>>>(u32_ptr(ctx, B200SPH_TAG) + o, n, tag);
    LAUNCH_CHECK();
    CU(cudaMemsetAsync(u32_ptr(ctx, B200SPH_PID) + o, 0, 4 * (size_t)n, ctx->stream));
    return 0;
}

// ---- mirror boundaries ----------------------------------------------------------------
// DomainManager(mirror_in_x ...) nnps_base.pyx:506-689: every particle within n_layers cells
// of a mirror plane gets an image on the other side (position reflected, the normal velocity
// component negated, everything else copied), images of images at the corners: x images
// first, then y images of the real particles AND of the x images, then z images of
// everything.  The reference re-selects at every update_domain; here the selection lives as
// long as the neighbour lists (its width covers the skin) and nnps_update refreshes the
// images' values in creation order before every evaluation.
static int mirror_refresh(b200sph_ctx *ctx)
{
    const HaloPtrs P = halo_ptrs(ctx);
    for (const auto &sg : ctx->mirror_segs) {
        if (sg.count == 0) continue;
        const ArrayInfo &ai = ctx->arr[sg.arr];
        const double plane2 = 2.0 * (sg.side == 0 ? ctx->dom_lo[sg.axis] : ctx->dom_hi[sg.axis]);
        k_mirror_copy<<<(unsigned)cdiv(sg.count, 256), 256, 0, ctx->stream>>>(P, ai.off, sg.idx, sg.count, ai.off + ai.n_real + sg.ghost_first, sg.axis, plane2);
        LAUNCH_CHECK();
    }
    particles_moved(ctx);
    return 0;
}

static int mirror_create(b200sph_ctx *ctx)
{
    int rc;
    if (elastic_allocated(ctx)) return set_err(ctx, "mirror boundaries: images carry the WCSPH fields only (x y z u v w rho h m), not the elastic-dynamics state");
    if ((rc = eos_flush(ctx))) return rc;
    // the cell size of the REAL particles decides the width (images have their sources' h)
    for (int a = 0; a < ctx->narr; a++) ctx->arr[a].n = ctx->arr[a].n_real;
    set_changed_with_h(ctx);
    ctx->mirror_built = false;
    if ((rc = b200sph_update_domain(ctx))) return rc;
    const double width = ctx->mirror_layers * ctx->cell_size * (1.0 + (ctx->force_kernel == 0 ? ctx->skin : 0.0));
    size_t nseg = 0;
    for (int a = 0; a < ctx->narr; a++) {
        for (int axis = 0; axis < 3; axis++) {
            if (!ctx->mirror[axis]) continue;
            // both sides select from the particles present BEFORE this axis (real + earlier axes' images)
            const int64_t n_sel = ctx->arr[a].n;
            for (int side = 0; side < 2; side++) {
                if (nseg == ctx->mirror_segs.size()) ctx->mirror_segs.emplace_back();
                b200sph_ctx::MirrorSeg &sg = ctx->mirror_segs[nseg++];
                sg.arr = a, sg.axis = axis, sg.side = side, sg.count = 0;
                ArrayInfo &ai = ctx->arr[a];
                sg.ghost_first = ai.n - ai.n_real;
                if (n_sel == 0) continue;
                const unsigned nb = (unsigned)cdiv(n_sel + 1, 256);
                k_flag_mirror<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X + axis), ai.off, n_sel, side == 0 ? ctx->dom_lo[axis] : ctx->dom_hi[axis], width, side, ctx->flag_a);
                LAUNCH_CHECK();
                if ((rc = device_scan(ctx, ctx->flag_a, ctx->flag_b, n_sel + 1))) return rc;
                uint32_t tot = 0;
                CU(cudaMemcpyAsync(&tot, ctx->flag_b + n_sel, 4, cudaMemcpyDeviceToHost, ctx->stream));
                CU(cudaStreamSynchronize(ctx->stream));
                if (tot == 0) continue;
                if ((rc = grow(ctx, sg.idx, tot, (size_t)tot + tot / 4 + 256))) return rc;
                k_save_idx<<<nb, 256, 0, ctx->stream>>>(n_sel, ctx->flag_a, ctx->flag_b, sg.idx);
                LAUNCH_CHECK();
                if ((rc = ensure_capacity(ctx, a, ai.n + tot))) return rc;   // may move the pool
                const int64_t o = ai.off + ai.n;
                // images arrive like ghosts, with tag = Ghost (2)
                if ((rc = arrival_init(ctx, o, tot, true, 2u))) return rc;
                k_mirror_copy<<<(unsigned)cdiv((int64_t)tot, 256), 256, 0, ctx->stream>>>(halo_ptrs(ctx), ai.off, sg.idx, (long long)tot, o, axis, 2.0 * (side == 0 ? ctx->dom_lo[axis] : ctx->dom_hi[axis]));
                LAUNCH_CHECK();
                sg.count = tot;
                ai.n += tot;
            }
        }
    }
    ctx->mirror_segs.resize(nseg);   // (a shrinking narr never happens; keeps the vector tidy)
    ctx->mirror_built = true;
    set_changed_with_h(ctx);
    return 0;
}

int b200sph_halo_layout(b200sph_ctx *ctx, int *halo_fields_out, int *migrate_fields_out)
{
    if (halo_fields_out) *halo_fields_out = halo_nf(ctx);
    if (migrate_fields_out) *migrate_fields_out = migrate_nf(ctx);
    return 0;
}

int b200sph_halo_pack(b200sph_ctx *ctx, int arr, int slot, double lo, double hi, double *dev_buf, int64_t cap, int64_t *count)
{
    if (int rcc = require_confirmed(ctx, "halo_pack")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "halo_pack: bad array %d", arr);
    const int64_t n = ctx->arr[arr].n_real, off = ctx->arr[arr].off;
    *count = 0;
    if (slot == 0 || slot == 1) ctx->halo_cnt[arr][slot] = 0;
    if (n == 0) return 0;
    const unsigned nb = (unsigned)cdiv(n + 1, 256);
    k_flag_range<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), off, n, lo, hi, 0, ctx->flag_a);
    LAUNCH_CHECK();
    if ((rc = device_scan(ctx, ctx->flag_a, ctx->flag_b, n + 1))) return rc;
    uint32_t tot = 0;
    CU(cudaMemcpyAsync(&tot, ctx->flag_b + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    *count = tot;
    if ((int64_t)tot > cap) return set_err(ctx, "halo_pack: %u particles selected but the buffer holds %lld", tot, (long long)cap);
    if (slot == 0 || slot == 1) {  // remember the selection for halo_pack_selected
        if ((rc = grow(ctx, ctx->halo_idx[arr][slot], tot, (size_t)tot + tot / 4 + 256))) return rc;
        ctx->halo_cnt[arr][slot] = tot;
        if (tot) {
            k_save_idx<<<nb, 256, 0, ctx->stream>>>(n, ctx->flag_a, ctx->flag_b, ctx->halo_idx[arr][slot]);
            LAUNCH_CHECK();
        }
    } else if (slot != -1) {
        return set_err(ctx, "halo_pack: slot must be -1, 0 or 1");
    }
    if (tot == 0) return 0;
    return with_halo_fields(ctx, [&](auto nf) {
        k_halo_gather_flag<decltype(nf)::value><<<nb, 256, 0, ctx->stream>>>(halo_ptrs(ctx), off, n, ctx->flag_a, ctx->flag_b, dev_buf, (long long)tot);
        LAUNCH_CHECK();
        return 0;
    });
}

int b200sph_halo_append(b200sph_ctx *ctx, int arr, const double *dev_buf, int64_t stride, int64_t n, int nfields, int as_real)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "halo_append: bad array %d", arr);
    const int hnf = halo_nf(ctx), mnf = migrate_nf(ctx);
    if (nfields != hnf && nfields != mnf) return set_err(ctx, "halo_append: nfields must be %d or %d", hnf, mnf);
    ArrayInfo &ai = ctx->arr[arr];
    if (as_real && ai.n != ai.n_real) return set_err(ctx, "halo_append(as_real): drop the ghosts of '%s' first (real particles must precede ghosts)", ai.name.c_str());
    if (n <= 0) return 0;
    if ((rc = ensure_capacity(ctx, arr, ai.n + n))) return rc;
    const int64_t o = ai.off + ai.n;
    const unsigned nb = (unsigned)cdiv(n, 256);
    // tag = Remote (1) for ghosts
    if ((rc = arrival_init(ctx, o, n, nfields == hnf, as_real ? 0u : 1u))) return rc;
    if (nfields == hnf) {
        rc = with_halo_fields(ctx, [&](auto nf) {
            k_halo_scatter<decltype(nf)::value><<<nb, 256, 0, ctx->stream>>>(halo_ptrs(ctx), o, dev_buf, stride, n);
            LAUNCH_CHECK();
            return 0;
        });
        if (rc) return rc;
    } else {
        for (int f = 0; f < mnf; f++) {
            const int p = migrate_msg[f];
            const double *src = dev_buf + (size_t)f * stride;
            const PropType t = prop_kind(p).type;
            if (t == PROP_F64) {
                CU(cudaMemcpyAsync(f64_ptr(ctx, p) + o, src, 8 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
                continue;
            }
            if (t == PROP_F32) k_f64_to_f32<<<nb, 256, 0, ctx->stream>>>(src, f32_ptr(ctx, p) + o, n);
            else k_f64_to_u32<<<nb, 256, 0, ctx->stream>>>(src, u32_ptr(ctx, p) + o, n);
            LAUNCH_CHECK();
        }
    }
    ai.n += n;
    if (as_real) ai.n_real += n;
    set_changed_with_h(ctx);
    return 0;
}

int b200sph_halo_pack_selected(b200sph_ctx *ctx, int arr, int slot, double *dev_buf, int64_t cap, int64_t *count)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (arr < 0 || arr >= ctx->narr || slot < 0 || slot > 1) return set_err(ctx, "halo_pack_selected: bad array / slot");
    const int64_t n = ctx->halo_cnt[arr][slot];
    *count = n;
    if (n > cap) return set_err(ctx, "halo_pack_selected: buffer too small");
    if (n == 0) return 0;
    return with_halo_fields(ctx, [&](auto nf) {
        k_halo_gather_idx<decltype(nf)::value><<<(unsigned)cdiv(n, 256), 256, 0, ctx->stream>>>(halo_ptrs(ctx), ctx->arr[arr].off, ctx->halo_idx[arr][slot], n, dev_buf);
        LAUNCH_CHECK();
        return 0;
    });
}

int b200sph_halo_overwrite(b200sph_ctx *ctx, int arr, int64_t ghost_first, const double *dev_buf, int64_t stride, int64_t n)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "halo_overwrite: bad array %d", arr);
    const ArrayInfo &ai = ctx->arr[arr];
    if (ghost_first < 0 || n < 0 || ai.n_real + ghost_first + n > ai.n)
        return set_err(ctx, "halo_overwrite: ghosts [%lld, %lld) outside the %lld ghosts of '%s'", (long long)ghost_first, (long long)(ghost_first + n), (long long)(ai.n - ai.n_real), ai.name.c_str());
    if (n == 0) return 0;
    const int64_t o = ai.off + ai.n_real + ghost_first;
    rc = with_halo_fields(ctx, [&](auto nf) {
        k_halo_scatter<decltype(nf)::value><<<(unsigned)cdiv(n, 256), 256, 0, ctx->stream>>>(halo_ptrs(ctx), o, dev_buf, stride, n);
        LAUNCH_CHECK();
        return 0;
    });
    if (rc) return rc;
    // values moved, the particle set did not: a light nnps_update is enough
    particles_moved(ctx);
    return 0;
}

int b200sph_nnps_drift(b200sph_ctx *ctx, double out[2])
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    out[0] = -1.0;
    out[1] = ctx->S_abs;
    if (!reusable_build(ctx)) return 0;
    if (retire_build(ctx)) return 0;
    if (ctx->n_sorted <= 0) { out[0] = 0.0; return 0; }
    if (!(ctx->packed_valid && ctx->drift_measured) && (rc = pack_positions_light(ctx, 2))) return rc;
    ctx->packed_valid = true, ctx->drift_measured = true;
    CU(cudaMemcpyAsync(ctx->red_u32_host, ctx->red_u32, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    out[0] = drift_need(ctx, ctx->red_u32_host);
    return 0;
}

// the ghost ranges [ghost_first[a], ghost_first[a] + counts[a]) of every array, checked against
// the array's ghosts, as the scatter's HaloAllArgs
static int ghost_ranges(b200sph_ctx *ctx, const int64_t *ghost_first, const int64_t *counts, HaloAllArgs &A)
{
    A.narr = ctx->narr;
    A.prefix[0] = 0;
    for (int a = 0; a < ctx->narr; a++) {
        const ArrayInfo &ai = ctx->arr[a];
        if (ghost_first[a] < 0 || counts[a] < 0 || ai.n_real + ghost_first[a] + counts[a] > ai.n)
            return set_err(ctx, "peer_recv: ghosts [%lld, %lld) outside the %lld ghosts of '%s'", (long long)ghost_first[a],
                           (long long)(ghost_first[a] + counts[a]), (long long)(ai.n - ai.n_real), ai.name.c_str());
        A.prefix[a + 1] = A.prefix[a] + counts[a];
        A.off[a] = ai.off + ai.n_real + ghost_first[a];
        A.idx[a] = nullptr;
    }
    return 0;
}

// ---- peer memory (same node, NVLink): staging buffers a neighbour rank writes into ----
int b200sph_ipc_alloc(b200sph_ctx *ctx, int64_t bytes, void **dev_ptr, void *handle64)
{
    CU(cudaSetDevice(ctx->device));
    void *p = nullptr;
    CU(cudaMalloc(&p, (size_t)std::max<int64_t>(bytes, 256)));
    CU(cudaMemset(p, 0, (size_t)std::max<int64_t>(bytes, 256)));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return set_err(ctx, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(handle64, &h, 64);
    *dev_ptr = p;
    return 0;
}

int b200sph_ipc_open(b200sph_ctx *ctx, const void *handle64, void **dev_ptr)
{
    CU(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    cudaError_t e = cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return set_err(ctx, "cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
    return 0;
}

int b200sph_ipc_close(b200sph_ctx *ctx, void *dev_ptr, int owner)
{
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (owner) CU(cudaFree(dev_ptr));
    else CU(cudaIpcCloseMemHandle(dev_ptr));
    return 0;
}

int b200sph_nnps_keep_build(b200sph_ctx *ctx)
{
    if (!reusable_build(ctx)) return set_err(ctx, "nnps_keep_build: there is no reusable neighbour build");
    ctx->drift_ok = true;
    return 0;
}

// ---- peer protocol (include/b200sph.h "peer protocol") ---------------------------------
// peer_publish / peer_send / peer_recv only RECORD what the epoch carries; peer_reduce
// launches the outgoing half as one k_peer_push and peer_end the incoming half as one
// k_peer_pull: two launches on the ghosts' critical path instead of seven dependent ones.
struct PeerPending {
    struct Dir { HaloAllArgs A; double *buf; unsigned long long *flag; long long tot; };
    Dir send[2], recv[2];
    int n_send = 0, n_recv = 0;
    int have_build = 0, with_dt = 0;
    bool publish = false;
    GhostPackArgs pack;
};
static void free_peer_pending(b200sph_ctx *ctx)
{
    delete ctx->pend;
    ctx->pend = nullptr;
}
static int peer_streams(b200sph_ctx *ctx)
{
    if (ctx->comm_stream) return 0;
    int lo = 0, hi = 0;
    CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));   // hi = the numerically lowest = highest priority
    CU(cudaStreamCreateWithPriority(&ctx->comm_stream, cudaStreamNonBlocking, hi));
    CU(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
    CU(cudaStreamCreateWithPriority(&ctx->red_stream, cudaStreamNonBlocking, hi));
    CU(cudaEventCreateWithFlags(&ctx->ev_pushed, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ctx->ev_red, cudaEventDisableTiming));
    CU(cudaEventRecord(ctx->ev_red, ctx->red_stream));
    ctx->pend = new PeerPending();
    return 0;
}

int b200sph_peer_init(b200sph_ctx *ctx, int rank, int world, void *handle64)
{
    CU(cudaSetDevice(ctx->device));
    if (world < 1 || world > B200SPH_MAX_RANKS || rank < 0 || rank >= world)
        return set_err(ctx, "peer_init: rank %d of %d (at most %d ranks)", rank, world, B200SPH_MAX_RANKS);
    if (ctx->peer_box) return set_err(ctx, "peer_init: already initialised");
    int rc = peer_streams(ctx);
    if (rc) return rc;
    const size_t boxes = cdiv(4096, sizeof(PeerBox));   // at least a page
    if ((rc = grow(ctx, ctx->peer_box, boxes, boxes)) || (rc = grow(ctx, ctx->peer_done, 2, 2)) ||
        (rc = grow(ctx, ctx->peer_dec_dev, 1, 1)) || (rc = grow(ctx, ctx->peer_dec_host, 1, 1)))
        return rc;
    CU(cudaMemset(ctx->peer_box, 0, boxes * sizeof(PeerBox)));
    CU(cudaMemset(ctx->peer_done, 0, 2 * sizeof(unsigned)));
    memset(ctx->peer_dec_host, 0, sizeof(PeerDecision));
    CU(cudaHostGetDevicePointer((void **)&ctx->peer_dec_hostdev, ctx->peer_dec_host, 0));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ctx->peer_box);
    if (e != cudaSuccess) return set_err(ctx, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    memcpy(handle64, &h, 64);
    ctx->peer_rank = rank;
    ctx->peer_world = world;
    ctx->peer_boxes[rank] = ctx->peer_box;
    return 0;
}

int b200sph_peer_connect(b200sph_ctx *ctx, const void *handles)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_box) return set_err(ctx, "peer_connect: call peer_init first");
    if (ctx->peer_connected) return 0;
    for (int r = 0; r < ctx->peer_world; r++) {
        if (r == ctx->peer_rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char *)handles + 64 * (size_t)r, 64);
        void *p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return set_err(ctx, "peer_connect: cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
        ctx->peer_boxes[r] = (PeerBox *)p;
    }
    ctx->peer_connected = true;
    return 0;
}

static PeerPtrs peer_ptrs(const b200sph_ctx *ctx)
{
    PeerPtrs R;
    for (int r = 0; r < B200SPH_MAX_RANKS; r++) R.box[r] = ctx->peer_boxes[r];
    return R;
}

int b200sph_peer_begin(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (!ctx->peer_connected) return set_err(ctx, "peer_begin: the mailboxes are not connected");
    if ((rc = eos_flush(ctx))) return rc;
    const int no_build = !reusable_build(ctx) || retire_build(ctx);
    if (!no_build && ctx->n_sorted > 0 && !(ctx->packed_valid && ctx->drift_measured) && (rc = pack_positions_light(ctx, 2)))
        return rc;
    if (!no_build) ctx->packed_valid = true, ctx->drift_measured = true;
    ctx->peer_epoch++;
    CU(cudaEventRecord(ctx->ev_fork, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->comm_stream, ctx->ev_fork, 0));
    if (ctx->profiling) {
        for (cudaEvent_t *e : {&ctx->halo_ev_fork, &ctx->halo_ev_chain, &ctx->halo_ev_sent, &ctx->halo_ev_reduced})
            if (!*e) {
                if (!ctx->ev_pool.empty()) { *e = ctx->ev_pool.back(); ctx->ev_pool.pop_back(); }
                else CU(cudaEventCreate(e));
            }
        CU(cudaEventRecord(ctx->halo_ev_fork, ctx->stream));
    }
    return no_build;
}

int b200sph_peer_publish(b200sph_ctx *ctx, int have_build, int with_dt)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_connected) return set_err(ctx, "peer_publish: the mailboxes are not connected");
    if (with_dt && !ctx->tc) return set_err(ctx, "peer_publish: no time-control block");
    ctx->pend->publish = true;
    ctx->pend->have_build = have_build && ctx->n_sorted > 0 ? 1 : (have_build ? 2 : 0);
    ctx->pend->with_dt = with_dt;
    ctx->pend->n_send = ctx->pend->n_recv = 0;
    return 0;
}

int b200sph_peer_send(b200sph_ctx *ctx, int slot, int nb_rank, int side, double *remote_staging, int64_t cap_doubles)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_connected) return set_err(ctx, "peer_send: the mailboxes are not connected");
    if (slot < -1 || slot > 1 || side < 0 || side > 1 || nb_rank < 0 || nb_rank >= ctx->peer_world || nb_rank == ctx->peer_rank)
        return set_err(ctx, "peer_send: bad slot / side / neighbour");
    HaloAllArgs A;
    A.narr = ctx->narr;
    A.prefix[0] = 0;
    for (int a = 0; a < ctx->narr; a++) {
        // slot -1: the flag alone (this rank has no reusable build: the neighbour must not wait)
        A.prefix[a + 1] = A.prefix[a] + (slot < 0 ? 0 : ctx->halo_cnt[a][slot]);
        A.off[a] = ctx->arr[a].off;
        A.idx[a] = slot < 0 ? nullptr : ctx->halo_idx[a][slot].p;
    }
    const int64_t tot = A.prefix[ctx->narr];
    if (tot * halo_nf(ctx) > cap_doubles) return set_err(ctx, "peer_send: staging buffer too small");
    if (!ctx->pend->publish) return set_err(ctx, "peer_send: peer_publish opens the outgoing half of an epoch");
    if (ctx->pend->n_send >= 2) return set_err(ctx, "peer_send: a slab has two neighbours");
    PeerPending::Dir &D = ctx->pend->send[ctx->pend->n_send++];
    D.A = A;
    D.buf = remote_staging;
    D.flag = &ctx->peer_boxes[nb_rank]->data_seq[ctx->peer_epoch & 1][side];
    D.tot = tot;
    return 0;
}

static void peer_dir(PeerDir &d, const PeerPending::Dir &p, unsigned *done)
{
    d.A = p.A;
    d.buf = p.buf;
    d.flag = p.flag;
    d.done = done;
    d.nblocks = (unsigned)cdiv(p.tot, PEER_NT);
}

// the outgoing half of the epoch: scalars + both messages, one launch
static int peer_push(b200sph_ctx *ctx)
{
    PeerPending &Q = *ctx->pend;
    if (!Q.publish) return set_err(ctx, "peer_reduce: nothing was published for this epoch");
    Q.publish = false;
    PeerPushArgs X;
    memset(&X, 0, sizeof(X));
    X.ndir = Q.n_send;
    for (int d = 0; d < Q.n_send; d++) peer_dir(X.d[d], Q.send[d], ctx->peer_done + d);
    X.rank = ctx->peer_rank;
    X.world = ctx->peer_world;
    X.have_build = Q.have_build;
    X.with_dt = Q.with_dt;
    X.kr = (float)ctx->radius_scale;
    X.S = (float)ctx->S_abs;
    X.red_u32 = ctx->red_u32;
    X.tc = ctx->tc;
    const unsigned blocks = 1 + X.d[0].nblocks + X.d[1].nblocks;
    return with_halo_fields(ctx, [&](auto nf) {
        k_peer_push<decltype(nf)::value><<<blocks, PEER_NT, 0, ctx->comm_stream>>>(halo_ptrs(ctx), X, peer_ptrs(ctx), ctx->peer_epoch);
        LAUNCH_CHECK();
        return 0;
    });
}

// the incoming half: both neighbours' messages scattered (and packed) by one launch
static int peer_pull(b200sph_ctx *ctx)
{
    PeerPending &Q = *ctx->pend;
    if (Q.n_recv == 0) return 0;
    PeerPullArgs X;
    memset(&X, 0, sizeof(X));
    X.ndir = Q.n_recv;
    for (int d = 0; d < Q.n_recv; d++) peer_dir(X.d[d], Q.recv[d], nullptr);
    Q.n_recv = 0;
    const unsigned blocks = X.d[0].nblocks + X.d[1].nblocks;
    return with_halo_fields(ctx, [&](auto nf) {
        k_peer_pull<decltype(nf)::value><<<blocks, PEER_NT, 0, ctx->comm_stream>>>(halo_ptrs(ctx), X, Q.pack, ctx->peer_epoch, ctx->peer_dec_hostdev);
        LAUNCH_CHECK();
        return 0;
    });
}

int b200sph_peer_reduce(b200sph_ctx *ctx, int with_dt)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_connected) return set_err(ctx, "peer_reduce: the mailboxes are not connected");
    int rc = peer_push(ctx);
    if (rc) return rc;
    if (ctx->profiling && ctx->halo_ev_sent) CU(cudaEventRecord(ctx->halo_ev_sent, ctx->comm_stream));
    CU(cudaEventRecord(ctx->ev_pushed, ctx->comm_stream));
    CU(cudaStreamWaitEvent(ctx->red_stream, ctx->ev_pushed, 0));   // my scalars are out before I wait for the others'
    k_peer_reduce<<<1, 32, 0, ctx->red_stream>>>(ctx->peer_box, ctx->peer_world, ctx->peer_epoch, 0, ctx->peer_dec_dev, ctx->peer_dec_hostdev,
                                                  ctx->tc, with_dt && ctx->tc ? 1 : 0);
    LAUNCH_CHECK();
    if (ctx->profiling && ctx->halo_ev_reduced) CU(cudaEventRecord(ctx->halo_ev_reduced, ctx->red_stream));
    CU(cudaEventRecord(ctx->ev_red, ctx->red_stream));
    return 0;
}

int b200sph_peer_recv(b200sph_ctx *ctx, int side, const int64_t *ghost_first, const int64_t *counts, const double *local_staging)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_connected) return set_err(ctx, "peer_recv: the mailboxes are not connected");
    if (side < 0 || side > 1) return set_err(ctx, "peer_recv: bad side");
    HaloAllArgs A;
    if (int rc = ghost_ranges(ctx, ghost_first, counts, A)) return rc;
    const int64_t tot = A.prefix[ctx->narr];
    if (tot == 0) return 0;
    int rc = refresh_ptype(ctx);
    if (rc) return rc;
    const bool repack = ctx->packed_valid && reusable_build(ctx) && ctx->n_sorted > 0;
    // the ghosts' state records too when the real particles' are in place (fused stage kernel;
    // WCSPH records: not with the elastic-dynamics arrays)
    const bool records = repack && ctx->state_packed && !elastic_allocated(ctx);
    GhostPackArgs R;
    memset(&R, 0, sizeof(R));
    R.rank = repack ? ctx->rank.p : nullptr;
    R.skey = ctx->skey;
    R.A = ctx->A; R.AB = ctx->AB;
    R.C = records ? ctx->C.p : nullptr;
    R.G = ctx->G;
    R.ptype = ctx->ptype;
    R.p = f32_ptr(ctx, B200SPH_P); R.cs = f32_ptr(ctx, B200SPH_CS);
    R.eos_any = ctx->spec_records && ctx->eos_last_valid ? 1 : 0;
    R.E = ctx->eos_last;
    if (ctx->pend->n_recv >= 2) return set_err(ctx, "peer_recv: a slab has two neighbours");
    PeerPending::Dir &D = ctx->pend->recv[ctx->pend->n_recv++];
    D.A = A;
    D.buf = const_cast<double *>(local_staging);
    D.flag = &ctx->peer_box->data_seq[ctx->peer_epoch & 1][side];
    D.tot = tot;
    ctx->pend->pack = R;          // the same for both sides: it describes the receiver
    ghosts_refreshed(ctx, repack, records);
    return 0;
}

int b200sph_peer_commit_dt(b200sph_ctx *ctx, double prev_factor, double new_factor, int adaptive, int advance, int snapshot_slot)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->comm_stream || !ctx->tc) return set_err(ctx, "peer_commit_dt: no epoch in flight / no time-control block");
    if (!(prev_factor > 0.0) || !(new_factor > 0.0)) return set_err(ctx, "peer_commit_dt: damping factors must be positive");
    if (snapshot_slot > 1) return set_err(ctx, "peer_commit_dt: snapshot slot must be 0 or 1");
    // behind the agreement (k_peer_reduce left the MIN in tc[2]), on its stream
    k_dt_commit<<<1, 1, 0, ctx->red_stream>>>(ctx->tc, prev_factor, new_factor, 1, adaptive, advance, ctx->t_final, ctx->t_eps);
    LAUNCH_CHECK();
    if (snapshot_slot >= 0) {
        CU(cudaMemcpyAsync(ctx->tc_host + 2 * snapshot_slot, ctx->tc, 2 * sizeof(double), cudaMemcpyDeviceToHost, ctx->red_stream));
        CU(cudaEventRecord(ctx->tc_evt[snapshot_slot], ctx->red_stream));
    }
    CU(cudaEventRecord(ctx->ev_red, ctx->red_stream));
    return 0;
}

int b200sph_peer_end(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->comm_stream) return set_err(ctx, "peer_end: no epoch in flight");
    if (ctx->pend->publish) return set_err(ctx, "peer_end: peer_reduce closes the outgoing half of an epoch");
    if (int rc = peer_pull(ctx)) return rc;
    if (ctx->profiling && ctx->halo_ev_chain) CU(cudaEventRecord(ctx->halo_ev_chain, ctx->comm_stream));
    CU(cudaEventRecord(ctx->ev_join, ctx->comm_stream));
    ctx->comm_pending = true;
    return 0;
}

int b200sph_peer_decision(b200sph_ctx *ctx, double *ratio_max)
{
    if (!ctx->peer_dec_host) return set_err(ctx, "peer_decision: no peer protocol");
    volatile PeerDecision *d = ctx->peer_dec_host;
    const unsigned long long want = ctx->peer_epoch;
    // the kernel that writes it is on the communication stream and needs no help from the host
    for (long long spin = 0; d->seq != want; spin++) {
        if ((spin & 0xFFFF) == 0xFFFF) {
            // nothing enqueued can be stuck for half a minute unless a peer died
            cudaError_t e = cudaStreamQuery(ctx->red_stream);
            if (e != cudaSuccess && e != cudaErrorNotReady) return set_err(ctx, "peer_decision: %s", cudaGetErrorString(e));
            if (e == cudaSuccess && d->seq != want) return set_err(ctx, "peer_decision: epoch %llu was never decided", want);
        }
    }
    if (d->error == want) return set_err(ctx, "peer protocol: a rank did not answer within %.0f s (epoch %llu)", PEER_TIMEOUT_NS * 1e-9, want);
    *ratio_max = d->value;
    if (d->value <= 1.0) {   // the skin controller's view of the build: the all-rank maximum (the same on every rank)
        ctx->drift_hist[0] = ctx->drift_hist[1];
        ctx->drift_hist[1] = d->value;
    }
    return 0;
}

int b200sph_peer_allreduce_dt(b200sph_ctx *ctx)
{
    CU(cudaSetDevice(ctx->device));
    if (!ctx->peer_connected) return set_err(ctx, "peer_allreduce_dt: the mailboxes are not connected");
    if (!ctx->tc) return set_err(ctx, "peer_allreduce_dt: no time-control block");
    ctx->peer_dt_epoch++;
    k_peer_publish<<<1, 32, 0, ctx->stream>>>(peer_ptrs(ctx), ctx->peer_rank, ctx->peer_world, ctx->peer_dt_epoch, 1, ctx->red_u32, 0.f, 0.f, 0, ctx->tc, 1);
    LAUNCH_CHECK();
    k_peer_reduce<<<1, 32, 0, ctx->stream>>>(ctx->peer_box, ctx->peer_world, ctx->peer_dt_epoch, 1, nullptr, nullptr, ctx->tc, 1);
    LAUNCH_CHECK();
    return 0;
}

int b200sph_drop_ghosts(b200sph_ctx *ctx, int arr)
{
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "drop_ghosts: bad array %d", arr);
    if (ctx->arr[arr].n != ctx->arr[arr].n_real) {
        CU(cudaSetDevice(ctx->device));
        if (int rci = materialise_pending(ctx)) return rci;
        ctx->arr[arr].n = ctx->arr[arr].n_real;
        set_changed(ctx);
    }
    return 0;
}

// Per-column particle counts for the slab re-cut.  Every thread walks COLUMN_RUN
// consecutive particles and merges equal bins before the atomic: particles are stored
// in cell order, so a run mostly stays in one column and the counters see ~n/32 atomics.
#define COLUMN_RUN 32
__global__ void k_column_counts(const double *__restrict__ x, long long off, long long n, double x0, double inv_w, int nbins,
                                unsigned long long *__restrict__ counts)
{
    const long long first = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * COLUMN_RUN;
    if (first >= n) return;
    const long long last = first + COLUMN_RUN < n ? first + COLUMN_RUN : n;
    int cur = -1;
    unsigned long long run = 0;
    for (long long i = first; i < last; i++) {
        int b = (int)floor((x[off + i] - x0) * inv_w);
        b = b < 0 ? 0 : (b >= nbins ? nbins - 1 : b);
        if (b != cur) {
            if (run) atomicAdd(&counts[cur], run);
            cur = b, run = 0;
        }
        run++;
    }
    if (run) atomicAdd(&counts[cur], run);
}

int b200sph_column_counts(b200sph_ctx *ctx, int arr, double x0, double inv_width, int nbins, unsigned long long *dev_counts)
{
    if (int rcc = require_confirmed(ctx, "column_counts")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "column_counts: bad array %d", arr);
    if (nbins < 1 || !(inv_width > 0.0) || !dev_counts) return set_err(ctx, "column_counts: bad bins");
    const ArrayInfo &ai = ctx->arr[arr];
    if (ai.n_real == 0) return 0;
    const unsigned nb = (unsigned)cdiv(cdiv(ai.n_real, COLUMN_RUN), 256);
    k_column_counts<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), ai.off, ai.n_real, x0, inv_width, nbins, dev_counts);
    LAUNCH_CHECK();
    return 0;
}

int b200sph_migrate_out(b200sph_ctx *ctx, int arr, double lo, double hi, double *dev_buf, int64_t cap, int64_t count[2])
{
    if (int rcc = require_confirmed(ctx, "migrate_out")) return rcc;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_pool(ctx);
    if (rc) return rc;
    if ((rc = eos_flush(ctx))) return rc;
    if (arr < 0 || arr >= ctx->narr) return set_err(ctx, "migrate_out: bad array %d", arr);
    ArrayInfo &ai = ctx->arr[arr];
    if (ai.n != ai.n_real) return set_err(ctx, "migrate_out: drop the ghosts of '%s' first", ai.name.c_str());
    const int64_t n = ai.n_real, off = ai.off;
    count[0] = count[1] = 0;
    if (n == 0) return 0;
    const unsigned nb = (unsigned)cdiv(n + 1, 256);
    const int mnf = migrate_nf(ctx);
    int64_t base = 0;  // doubles written so far
    for (int side = 0; side < 2; side++) {
        k_flag_range<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), off, n, lo, hi, side == 0 ? 1 : 2, ctx->flag_a);
        LAUNCH_CHECK();
        if ((rc = device_scan(ctx, ctx->flag_a, ctx->flag_b, n + 1))) return rc;
        uint32_t tot = 0;
        CU(cudaMemcpyAsync(&tot, ctx->flag_b + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        count[side] = tot;
        if (base + (int64_t)tot * mnf > cap * mnf) return set_err(ctx, "migrate_out: buffer too small");
        for (int f = 0; tot && f < mnf; f++) {
            const int p = migrate_msg[f];
            const long long at = base + (long long)f * tot;
            const PropType t = prop_kind(p).type;
            if (t == PROP_F64) k_gather_f64<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, p), off, n, ctx->flag_a, ctx->flag_b, dev_buf, at);
            else if (t == PROP_F32) k_gather_f32_as_f64<<<nb, 256, 0, ctx->stream>>>(f32_ptr(ctx, p), off, n, ctx->flag_a, ctx->flag_b, dev_buf, at);
            else k_gather_u32_as_f64<<<nb, 256, 0, ctx->stream>>>(u32_ptr(ctx, p), off, n, ctx->flag_a, ctx->flag_b, dev_buf, at);
            LAUNCH_CHECK();
        }
        base += (int64_t)tot * mnf;
    }
    if (count[0] + count[1] == 0) return 0;
    // stable compaction of the keepers, property by property, through the staging buffer
    k_flag_range<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, B200SPH_X), off, n, lo, hi, 3, ctx->flag_a);
    LAUNCH_CHECK();
    if ((rc = device_scan(ctx, ctx->flag_a, ctx->flag_b, n + 1))) return rc;
    const int64_t keep = n - count[0] - count[1];
    if ((rc = ensure_stage(ctx, n))) return rc;
    // the keepers keep what the migration message carries, and tag and pid (the other fp32
    // fields are recomputed); 4-byte properties move as bits
    for (int f = 0; f < mnf + 2; f++) {
        const int p = f < mnf ? migrate_msg[f] : (f == mnf ? B200SPH_TAG : B200SPH_PID);
        const size_t esz = prop_kind(p).size();
        if (esz == 8) k_gather_f64<<<nb, 256, 0, ctx->stream>>>(f64_ptr(ctx, p), off, n, ctx->flag_a, ctx->flag_b, ctx->stage_buf, 0);
        else k_gather_u32<<<nb, 256, 0, ctx->stream>>>(u32_ptr(ctx, p), off, n, ctx->flag_a, ctx->flag_b, (uint32_t *)ctx->stage_buf.p);
        LAUNCH_CHECK();
        if (keep) CU(cudaMemcpyAsync((char *)ctx->prop[p] + esz * (size_t)off, ctx->stage_buf, esz * (size_t)keep, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    ai.n = ai.n_real = keep;
    set_changed_with_h(ctx);
    return 0;
}

int b200sph_get_stats(b200sph_ctx *ctx, b200sph_stats *out)
{
    if (!ctx->pending.empty()) {
        CU(cudaSetDevice(ctx->device));
        CU(cudaStreamSynchronize(ctx->stream));
        for (auto &pe : ctx->pending) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, pe.e0, pe.e1);
            if (pe.slot == 0) ctx->stats.ms_nnps += ms;
            else if (pe.slot == 1) ctx->stats.ms_pair += ms;
            else ctx->stats.ms_other += ms;
            ctx->ev_pool.push_back(pe.e0);
            ctx->ev_pool.push_back(pe.e1);
        }
        ctx->pending.clear();
    }
    if (!ctx->halo_pending.empty()) {
        CU(cudaSetDevice(ctx->device));
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->comm_stream) CU(cudaStreamSynchronize(ctx->comm_stream));
        if (ctx->red_stream) CU(cudaStreamSynchronize(ctx->red_stream));
        for (auto &h : ctx->halo_pending) {
            float a = 0.f, b = 0.f;
            cudaEventElapsedTime(&a, h.fork, h.chain);
            cudaEventElapsedTime(&b, h.fork, h.end);
            ctx->stats.ms_halo_chain += a;
            ctx->stats.ms_pair_wall += b;
            if (h.sent && h.reduced) {
                float c = 0.f, d = 0.f;
                if (cudaEventElapsedTime(&c, h.fork, h.sent) == cudaSuccess) ctx->stats.ms_halo_sent += c;
                if (cudaEventElapsedTime(&d, h.fork, h.reduced) == cudaSuccess) ctx->stats.ms_halo_reduced += d;
                ctx->ev_pool.push_back(h.sent); ctx->ev_pool.push_back(h.reduced);
            }
            ctx->ev_pool.push_back(h.fork); ctx->ev_pool.push_back(h.chain); ctx->ev_pool.push_back(h.end);
        }
        ctx->halo_pending.clear();
    }
    ctx->stats.full_builds = ctx->n_full_builds;
    ctx->stats.light_updates = ctx->n_light_updates;
    ctx->stats.list_builds = ctx->n_list_builds;
    ctx->stats.list_entries_per_particle = ctx->capg;
    ctx->stats.deferred_failed = ctx->n_deferred_failed;
    ctx->stats.fused_stages = ctx->n_fused;
    ctx->stats.overlapped = ctx->n_overlapped;
    ctx->stats.proactive_builds = ctx->n_proactive;
    ctx->stats.chunks_interior = ctx->chunks_valid ? ctx->n_chunk_interior : 0;
    ctx->stats.chunks_boundary = ctx->chunks_valid ? ctx->n_chunk_boundary : 0;
    *out = ctx->stats;
    return 0;
}
int b200sph_reset_stats(b200sph_ctx *ctx)
{
    b200sph_stats tmp;
    b200sph_get_stats(ctx, &tmp);  // drain pending events
    memset(&ctx->stats, 0, sizeof(ctx->stats));
    ctx->n_full_builds = ctx->n_light_updates = ctx->n_list_builds = ctx->n_deferred_failed = ctx->n_fused = ctx->n_overlapped = ctx->n_proactive = ctx->n_pair_r32 = 0;
    ctx->n_half_materialised = 0;
    return 0;
}
int b200sph_half_materialised(b200sph_ctx *ctx, int64_t *out)
{
    *out = ctx->n_half_materialised;
    return 0;
}
int b200sph_records32_launches(b200sph_ctx *ctx, int64_t *out)
{
    *out = ctx->n_pair_r32;
    return 0;
}
int b200sph_set_async_copies(b200sph_ctx *ctx, int on)
{
    ctx->async_copies = on != 0;
    if (!on) CU(cudaStreamSynchronize(ctx->stream));
    return 0;
}
int b200sph_set_profiling(b200sph_ctx *ctx, int on)
{
    ctx->profiling = on < 0 ? 0 : (on > 2 ? 1 : on);
    return 0;
}

}  // extern "C"
