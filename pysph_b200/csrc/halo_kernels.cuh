// halo_kernels.cuh -- halo / migration kernels of the slab decomposition.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// halo / migration kernels
// --------------------------------------------------------------------------
// mode 0: flag = lo <= x < hi ; mode 1: flag = x < lo ; mode 2: flag = x >= hi ;
// mode 3: flag = keep (lo <= x < hi)
__global__ void k_flag_range(const double *__restrict__ x, long long off, long long n, double lo,
                             double hi, int mode, uint32_t *__restrict__ flag)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    uint32_t f = 0;
    if (i < n) {
        const double v = x[off + i];
        if (mode == 0 || mode == 3) f = (v >= lo && v < hi);
        else if (mode == 1) f = v < lo;
        else f = v >= hi;
    }
    flag[i] = f;  // flag[n] = 0 so that scan[n] = total
}

__global__ void k_gather_f64(const double *__restrict__ src, long long off, long long n,
                             const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                             double *__restrict__ dst, long long dst_off)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flag[i]) dst[dst_off + pos[i]] = src[off + i];
}
__global__ void k_gather_u32_as_f64(const uint32_t *__restrict__ src, long long off, long long n,
                                    const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                                    double *__restrict__ dst, long long dst_off)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flag[i]) dst[dst_off + pos[i]] = (double)src[off + i];
}
__global__ void k_gather_u32(const uint32_t *__restrict__ src, long long off, long long n,
                             const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                             uint32_t *__restrict__ dst)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flag[i]) dst[pos[i]] = src[off + i];
}
// the ghost message: B200SPH_HALO_FIELDS (x y z u v w rho h m), or with the elastic-dynamics
// arrays allocated B200SPH_HALO_FIELDS_SOLID (+ s00 s01 s02 s11 s12 s22 and, last, the fp32
// property cs widened to a double: no equation of that scheme recomputes it); NF is a
// template parameter so that the 9-field kernels stay the unrolled ones that were measured
#define HALO_ND(NF) ((NF) == B200SPH_HALO_FIELDS ? B200SPH_HALO_FIELDS : B200SPH_HALO_FIELDS_SOLID - 1)
struct HaloPtrs {
    double *p[B200SPH_HALO_FIELDS_SOLID - 1];
    float *cs;
};
// all NF fields of the selected particles in one launch (field-major, tight)
template <int NF>
__global__ void k_halo_gather_flag(HaloPtrs P, long long off, long long n, const uint32_t *__restrict__ flag,
                                   const uint32_t *__restrict__ pos, double *__restrict__ dst, long long tot)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flag[i]) return;
    const long long k = pos[i];
#pragma unroll
    for (int f = 0; f < HALO_ND(NF); f++) dst[(long long)f * tot + k] = P.p[f][off + i];
    if (NF != B200SPH_HALO_FIELDS) dst[(long long)(NF - 1) * tot + k] = (double)P.cs[off + i];
}
template <int NF>
__global__ void k_halo_gather_idx(HaloPtrs P, long long off, const uint32_t *__restrict__ idx, long long n,
                                  double *__restrict__ dst)
{
    long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long i = idx[k];
#pragma unroll
    for (int f = 0; f < HALO_ND(NF); f++) dst[(long long)f * n + k] = P.p[f][off + i];
    if (NF != B200SPH_HALO_FIELDS) dst[(long long)(NF - 1) * n + k] = (double)P.cs[off + i];
}
template <int NF>
__global__ void k_halo_scatter(HaloPtrs P, long long o, const double *__restrict__ src, long long stride, long long n)
{
    long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
#pragma unroll
    for (int f = 0; f < HALO_ND(NF); f++) P.p[f][o + k] = src[(long long)f * stride + k];
    if (NF != B200SPH_HALO_FIELDS) P.cs[o + k] = (float)src[(long long)(NF - 1) * stride + k];
}
// mirror images (nnps_base.pyx:506-689): side 0: (v - plane) <= width, side 1: (plane - v) <= width
__global__ void k_flag_mirror(const double *__restrict__ v, long long off, long long n, double plane, double width, int side,
                              uint32_t *__restrict__ flag)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    uint32_t f = 0;
    if (i < n) {
        const double x = v[off + i];
        f = side == 0 ? ((x - plane) <= width) : ((plane - x) <= width);
    }
    flag[i] = f;  // flag[n] = 0 so that scan[n] = total
}
// image k = source idx[k] reflected in the plane normal to `axis`: position 2 plane - x, the
// normal velocity component negated, the other fields of the ghost message copied
__global__ void k_mirror_copy(HaloPtrs P, long long off, const uint32_t *__restrict__ idx, long long n, long long dst,
                              int axis, double plane2)
{
    long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long i = off + idx[k];
#pragma unroll
    for (int f = 0; f < B200SPH_HALO_FIELDS; f++) {
        double v = P.p[f][i];
        if (f == axis) v = plane2 - v;
        else if (f == 3 + axis) v = -v;
        P.p[f][dst + k] = v;
    }
}
__global__ void k_save_idx(long long n, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                           uint32_t *__restrict__ idx)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flag[i]) idx[pos[i]] = (uint32_t)i;
}
__global__ void k_f64_to_u32(const double *__restrict__ in, uint32_t *__restrict__ out, long long n)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint32_t)in[i];
}
__global__ void k_gather_f32_as_f64(const float *__restrict__ src, long long off, long long n,
                                    const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                                    double *__restrict__ dst, long long dst_off)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (flag[i]) dst[dst_off + pos[i]] = (double)src[off + i];
}
__global__ void k_fill_u32(uint32_t *p, long long n, uint32_t v)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// --------------------------------------------------------------------------
// Peer protocol: the ghost refresh of an evaluation and the scalar agreement that goes
// with it (is every rank's neighbour build still valid?  the global time step) without a
// library collective.  Every rank owns a MAILBOX in device memory that the other ranks of
// the node write into over NVLink (cudaIpc mappings):
//   scal[parity][r]  {drift ratio, dt proposal, epoch}   written by rank r, read by me
//   data_seq[parity][side]   epoch of the halo message my left / right neighbour has
//                            finished writing into my staging buffer
// Writers store the payload, __threadfence_system(), then the epoch; readers poll the
// epoch with volatile loads and read the payload behind it.  Slots are double buffered by
// epoch parity: a rank can only be two epochs ahead of the slowest one, because passing
// epoch e needs every rank's epoch-e flags, which they publish after finishing e - 1.
// The kernels are a few small CTAs on a high-priority stream, so they are scheduled as
// soon as any CTA of the concurrently running interior pair kernel retires.
// A wait that lasts longer than PEER_TIMEOUT_NS sets the error word and carries on (the
// host then raises): a dead peer must not hang the GPU.
// --------------------------------------------------------------------------
#define PEER_TIMEOUT_NS 20000000000ull
struct PeerSlot {
    double v[2];
    unsigned long long seq, pad;
};
struct PeerBox {
    PeerSlot scal[2][B200SPH_MAX_RANKS];   // refresh epochs
    PeerSlot dts[2][B200SPH_MAX_RANKS];    // stand-alone time-step agreement (own epoch counter)
    unsigned long long data_seq[2][2];
};
struct PeerPtrs {
    PeerBox *box[B200SPH_MAX_RANKS];       // box[r]: rank r's mailbox (own rank: the local one)
};
struct PeerDecision {                      // pinned, mapped host memory
    double value;
    unsigned long long seq;
    unsigned long long error;
};

__device__ __forceinline__ bool peer_wait(const volatile unsigned long long *flag, unsigned long long want)
{
    if (*flag == want) return true;
    const unsigned long long t0 = peer_now_ns();
    unsigned ns = 32;
    while (*flag != want) {
        __nanosleep(ns);
        if (ns < 1024) ns *= 2;
        if (peer_now_ns() - t0 > PEER_TIMEOUT_NS) return false;
    }
    return true;
}

// the used-up fraction of the neighbour-list skin S: (2 |dx|max + k dh) / S from the drift
// that k_pack_pos_light / the fused stage kernel max-reduced into red_u32[0..1] (|dx|^2 and
// dh as fp32 bits); 2 (= expired) without a skin
__device__ __forceinline__ double drift_ratio(const unsigned *__restrict__ red_u32, float kr, float S)
{
    const float need = 2.0f * sqrtf(__uint_as_float(red_u32[0])) + kr * __uint_as_float(red_u32[1]);
    return S > 0.f ? (double)(need / S) : 2.0;
}

// this rank's scalars into the slot `sl` of one rank's mailbox: v0 = the drift ratio, 2 = no
// reusable build (have_build 0), 0 = a rank without particles (have_build 2); v1 = the dt
// proposal tc[2] (with_dt) or +inf
__device__ __forceinline__ void peer_publish_slot(PeerSlot *sl, unsigned long long epoch, const unsigned *__restrict__ red_u32,
                                                  float kr, float S, int have_build, const double *__restrict__ tc, int with_dt)
{
    double v0 = 2.0;                 // have_build == 0: no reusable build
    if (have_build == 1) {
        v0 = drift_ratio(red_u32, kr, S);
    } else if (have_build == 2) {
        v0 = 0.0;                    // a rank without particles keeps whatever the others keep
    }
    const double v1 = with_dt ? tc[2] : __longlong_as_double(0x7ff0000000000000LL);
    sl->v[0] = v0;
    sl->v[1] = v1;
    __threadfence_system();
    *(volatile unsigned long long *)&sl->seq = epoch;
}

// lane r publishes this rank's scalars to rank r.  which = 0: refresh epoch, which = 1: the
// stand-alone time-step agreement (v1 = dt proposal).
__global__ void k_peer_publish(PeerPtrs R, int rank, int world, unsigned long long epoch, int which,
                               const unsigned *__restrict__ red_u32, float kr, float S, int have_build,
                               const double *__restrict__ tc, int with_dt)
{
    const int r = threadIdx.x;
    if (r >= world) return;
    PeerSlot *sl = which == 0 ? &R.box[r]->scal[epoch & 1][rank] : &R.box[r]->dts[epoch & 1][rank];
    peer_publish_slot(sl, epoch, red_u32, kr, S, have_build, tc, with_dt);
}

// wait for every rank's scalars of this epoch: MAX of v0 -> decision (device + host),
// MIN of v1 -> tc[2] when with_dt
__global__ void k_peer_reduce(PeerBox *mine, int world, unsigned long long epoch, int which, double *__restrict__ dec_dev,
                              PeerDecision *dec_host, double *__restrict__ tc, int with_dt)
{
    const int r = threadIdx.x;
    double v0 = -1e300, v1 = __longlong_as_double(0x7ff0000000000000LL);
    bool ok = true;
    if (r < world) {
        PeerSlot *sl = which == 0 ? &mine->scal[epoch & 1][r] : &mine->dts[epoch & 1][r];
        ok = peer_wait(&sl->seq, epoch);
        __threadfence_system();
        v0 = *(volatile double *)&sl->v[0];
        v1 = *(volatile double *)&sl->v[1];
    }
    const unsigned bad = __ballot_sync(0xffffffffu, !ok);
    for (int o = 16; o > 0; o >>= 1) {
        v0 = fmax(v0, __shfl_xor_sync(0xffffffffu, v0, o));
        v1 = fmin(v1, __shfl_xor_sync(0xffffffffu, v1, o));
    }
    if (r == 0) {
        if (bad) v0 = 1e30;          // a rank never answered: nobody may trust its lists
        if (dec_dev) dec_dev[0] = v0;
        if (with_dt && tc) tc[2] = v1;
        if (dec_host) {
            if (bad) dec_host->error = epoch;
            dec_host->value = v0;
            __threadfence_system();
            *(volatile unsigned long long *)&dec_host->seq = epoch;
        }
    }
}

// The refresh message of ALL arrays: the block of array a starts at NF * prefix[a] doubles,
// field-major and tight inside the block.
struct HaloAllArgs {
    int narr;
    long long prefix[B200SPH_MAX_ARRAYS + 1];  // particles before array a in the message
    long long off[B200SPH_MAX_ARRAYS];         // pool offset of the first particle addressed
    const uint32_t *idx[B200SPH_MAX_ARRAYS];   // gather: saved selection (relative to off); scatter: unused
};
// entry k (< prefix[narr]) of the message: array a, its r-th particle of cnt
__device__ __forceinline__ int halo_entry(const HaloAllArgs &A, long long k, long long &r, long long &cnt)
{
    int a = 0;
    while (k >= A.prefix[a + 1]) a++;
    r = k - A.prefix[a];
    cnt = A.prefix[a + 1] - A.prefix[a];
    return a;
}
// entry k gathered from the pool into the message at dst (a peer pointer: the neighbour's
// staging buffer)
template <int NF>
__device__ __forceinline__ void halo_gather_entry(const HaloPtrs &P, const HaloAllArgs &A, long long k, double *__restrict__ dst)
{
    long long r, cnt;
    const int a = halo_entry(A, k, r, cnt);
    const long long i = A.off[a] + A.idx[a][r];
    double *out = dst + NF * A.prefix[a] + r;
#pragma unroll
    for (int f = 0; f < HALO_ND(NF); f++) out[(long long)f * cnt] = P.p[f][i];
    if (NF != B200SPH_HALO_FIELDS) out[(long long)(NF - 1) * cnt] = (double)P.cs[i];
}

// the packed pair records of a ghost, written by the receiving kernel (the fused stage
// kernel only packs real particles): {A, B} at its sorted slot and C with the equation of
// state that the last evaluation applied to ghosts (eos_tab_eval, state_record)
struct GhostPackArgs {
    const uint32_t *rank, *skey;   // rank == nullptr: no records (no reusable build)
    float4 *A, *AB, *C;            // C == nullptr: positions only
    GridDev G;
    const uint8_t *ptype;
    const float *p, *cs;
    int eos_any;
    EosTab E;
};
// entry k of the message at src (written by the peer: read past L1) scattered over its ghost
// in place, and with a valid neighbour build the ghost's packed records refreshed in the
// same pass (x, y, z, h are fields 0, 1, 2, 7)
template <int NF>
__device__ __forceinline__ void halo_scatter_entry(const HaloPtrs &P, const HaloAllArgs &A, long long k, const double *src,
                                                   const GhostPackArgs &R)
{
    long long r, cnt;
    const int a = halo_entry(A, k, r, cnt);
    const double *in = src + NF * A.prefix[a] + r;
    const long long g = A.off[a] + r;
    double v[HALO_ND(NF)];
#pragma unroll
    for (int f = 0; f < HALO_ND(NF); f++) {
        v[f] = __ldcg(in + (long long)f * cnt);
        P.p[f][g] = v[f];
    }
    if (NF != B200SPH_HALO_FIELDS) P.cs[g] = (float)__ldcg(in + (long long)(NF - 1) * cnt);
    if (R.rank) {
        const uint32_t s = R.rank[g];
        const float4 q = pack_position(R.G, R.skey[s], v[0], v[1], v[2], v[7]);
        R.A[s] = q;
        R.AB[2 * (size_t)s] = q;
        if (R.C) {
            // fields: 0..2 x y z, 3..5 u v w, 6 rho, 7 h, 8 m
            const int t = (int)R.ptype[g];
            const int ar = t & 7;
            double rr = v[6];
            float pg, csg;
            if (R.eos_any && R.E.on[ar] && !R.E.real_only[ar]) {
                eos_tab_eval(R.E, ar, rr, pg, csg);   // the record only; the pool side follows with the EOS calls
            } else {
                pg = R.p[g];
                csg = R.cs[g];
            }
            float4 b, c;
            state_record(v[3], v[4], v[5], v[8], rr, pg, csg, t, b, c);
            R.AB[2 * (size_t)s + 1] = b;
            R.C[s] = c;
        }
    }
}

// One direction of the fused push / pull kernels below.
struct PeerDir {
    HaloAllArgs A;
    double *buf;                 // push: the neighbour's staging buffer (peer pointer); pull: mine
    unsigned long long *flag;    // push: data_seq in the neighbour's mailbox; pull: in mine
    unsigned *done;              // push: block counter of this direction
    unsigned nblocks;            // blocks of PEER_NT messages entries (0: the flag alone)
};
#define PEER_NT 256
struct PeerPushArgs {
    PeerDir d[2];
    int ndir;
    // the scalars of k_peer_publish, sent by block 0
    int rank, world, have_build, with_dt;
    float kr, S;
    const unsigned *red_u32;
    const double *tc;
};

// The outgoing half of a refresh epoch in ONE launch: block 0 publishes this rank's scalars
// to every mailbox and raises the flag of a direction that has nothing to carry; the other
// blocks gather the messages into the neighbours' staging buffers, and whichever block of a
// direction finishes last raises that neighbour's data-ready flag (every block fences its
// stores first).
template <int NF>
__global__ void __launch_bounds__(PEER_NT) k_peer_push(HaloPtrs P, PeerPushArgs X, PeerPtrs R, unsigned long long epoch)
{
    if (blockIdx.x == 0) {
        const int r = threadIdx.x;
        if (r < X.world) {
            peer_publish_slot(&R.box[r]->scal[epoch & 1][X.rank], epoch, X.red_u32, X.kr, X.S, X.have_build, X.tc, X.with_dt);
        } else if (r >= 32 && r < 32 + X.ndir && X.d[r - 32].nblocks == 0) {
            __threadfence_system();
            *(volatile unsigned long long *)X.d[r - 32].flag = epoch;
        }
        return;
    }
    const unsigned b = blockIdx.x - 1;
    const int d = b >= X.d[0].nblocks ? 1 : 0;
    const PeerDir &D = X.d[d];
    const long long k = (long long)(b - (d ? X.d[0].nblocks : 0u)) * PEER_NT + threadIdx.x;
    if (k < D.A.prefix[D.A.narr]) halo_gather_entry<NF>(P, D.A, k, D.buf);
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(D.done, 1u);
        if (prev == D.nblocks - 1) {
            *D.done = 0;                     // re-armed for the next launch on this stream
            __threadfence_system();
            *(volatile unsigned long long *)D.flag = epoch;
        }
    }
}

struct PeerPullArgs {
    PeerDir d[2];
    int ndir;
};
// The incoming half in ONE launch: both neighbours' messages scattered over the ghosts, every
// block behind the data-ready flag of its own direction (a block of the left message does
// not wait for the right neighbour).
template <int NF>
__global__ void __launch_bounds__(PEER_NT) k_peer_pull(HaloPtrs P, PeerPullArgs X, GhostPackArgs R, unsigned long long epoch,
                                                       PeerDecision *dec_host)
{
    __shared__ int s_ok;
    const int d = blockIdx.x >= X.d[0].nblocks ? 1 : 0;
    const PeerDir &D = X.d[d];
    if (threadIdx.x == 0) {
        s_ok = peer_wait((const volatile unsigned long long *)D.flag, epoch) ? 1 : 0;
        __threadfence_system();
    }
    __syncthreads();
    if (!s_ok) {
        if (threadIdx.x == 0 && dec_host) dec_host->error = epoch;
        return;
    }
    const long long k = (long long)(blockIdx.x - (d ? X.d[0].nblocks : 0u)) * PEER_NT + threadIdx.x;
    if (k >= D.A.prefix[D.A.narr]) return;
    halo_scatter_entry<NF>(P, D.A, k, D.buf, R);
}

// ---- interior / boundary split of the list consumer ---------------------------------------
// sflag[s] = 1 if the particle at sorted slot s is a ghost
__global__ void k_sorted_ghost_flag(const uint8_t *__restrict__ ptype, const uint32_t *__restrict__ perm, long long n,
                                    uint8_t *__restrict__ sflag)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) sflag[s] = (ptype[perm[s]] & PT_GHOST) ? 1 : 0;
}
// chunk = LIST_NT consecutive destinations = one CTA of the list consumers.  A chunk is a
// BOUNDARY chunk if a ghost is among its destinations or in one of their lists: it has to
// wait for the halo; the others can run while the halo is in flight.
__global__ void __launch_bounds__(LIST_NT) k_chunk_classify(const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ lst,
                                                           const int capg, const uint8_t *__restrict__ sflag, long long n,
                                                           uint32_t *__restrict__ chunk_flag)
{
    const long long s = (long long)blockIdx.x * LIST_NT + threadIdx.x;
    int hit = 0;
    if (s < n) {
        hit = sflag[s];
        const int count = (int)cnt[s];
        const uint32_t *my = list_slot(lst, capg, s);
        for (int k = 0; k < count && !hit; k++) hit = sflag[LIST_J(my[(size_t)k * 32u])];
    }
    __shared__ int s_hit;
    if (threadIdx.x == 0) s_hit = 0;
    __syncthreads();
    if (hit) s_hit = 1;
    __syncthreads();
    if (threadIdx.x == 0) chunk_flag[blockIdx.x] = s_hit ? 1u : 0u;
    if (blockIdx.x == 0 && threadIdx.x == 0) chunk_flag[gridDim.x] = 0u;   // so that scan[nchunks] = total
}
__global__ void k_chunk_split(long long nchunks, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                              uint32_t *__restrict__ boundary, uint32_t *__restrict__ interior)
{
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    if (flag[c]) boundary[pos[c]] = (uint32_t)c;
    else interior[c - pos[c]] = (uint32_t)c;
}
