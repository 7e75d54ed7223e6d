// cuda_shim.h -- TEST INFRASTRUCTURE.  A minimal host stand-in for <cuda_runtime.h> and the
// CUDA device intrinsics csrc/b200sph.cu uses, so that the WHOLE library (host C-ABI code +
// kernels, transformed by tests/cpu_emul/transform.py: launches `k<<<g,b,s,st>>>(args)` become
// emu::launch(...) calls) can be compiled with g++ and run without a GPU.  "Device" memory is
// host memory; a launch runs its blocks one after another, the threads of a block either one
// after another (kernels without intra-block communication), or as lock-stepped OS threads with
// real __syncthreads / warp shuffles / ballots / atomics.  It is slow and proves nothing about
// performance, occupancy or memory spaces -- it checks that the code computes the right thing.
#pragma once
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

// ---- vector types ------------------------------------------------------------------------
struct float4 { float x, y, z, w; };
struct float2 { float x, y; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
struct idx3 { unsigned x, y, z; };

// ---- qualifiers ----------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static

namespace emu {
void yield();   // cuda_shim.cpp: hand the core to the next lock-stepped lane
struct Barrier {
    int n;
    std::atomic<int> arrived{0};
    std::atomic<int> phase{0};
    explicit Barrier(int n_) : n(n_) {}
    void wait()
    {
        const int ph = phase.load(std::memory_order_acquire);
        if (arrived.fetch_add(1, std::memory_order_acq_rel) == n - 1) {
            arrived.store(0, std::memory_order_relaxed);
            phase.store(ph + 1, std::memory_order_release);
        } else {
            while (phase.load(std::memory_order_acquire) == ph) emu::yield();
        }
    }
};
struct WarpCtx {
    Barrier bar{32};
    unsigned long long slot[32];
};
struct BlockCtx {
    Barrier bar;
    std::vector<WarpCtx> warps;
    explicit BlockCtx(int nt) : bar(nt), warps((size_t)(nt + 31) / 32) {}
};
extern thread_local idx3 t_threadIdx, t_blockIdx, t_blockDim, t_gridDim;
extern thread_local WarpCtx *t_warp;     // non-null: lanes run in lock step (fibers, or real threads)
extern thread_local BlockCtx *t_block;   // non-null: the block's threads run in lock step
extern thread_local int t_lane;
enum Mode { SEQ = 0, WARP = 1, BLOCK = 2 };
void launch(long long grid, long long block, int mode, const std::function<void()> &body);
template <class T> static inline unsigned long long to_bits(T v) { unsigned long long b = 0; memcpy(&b, &v, sizeof(T)); return b; }
template <class T> static inline T from_bits(unsigned long long b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
template <class T> static inline T warp_read(T v, int src, bool valid)
{
    if (!t_warp) return v;
    t_warp->slot[t_lane] = to_bits(v);
    t_warp->bar.wait();
    const T r = valid ? from_bits<T>(t_warp->slot[src & 31]) : v;
    t_warp->bar.wait();
    return r;
}
}  // namespace emu
#define threadIdx emu::t_threadIdx
#define blockIdx emu::t_blockIdx
#define blockDim emu::t_blockDim
#define gridDim emu::t_gridDim

// ---- synchronisation / warp intrinsics ---------------------------------------------------------
static inline void __syncthreads() { if (emu::t_block) emu::t_block->bar.wait(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { if (emu::t_warp) emu::t_warp->bar.wait(); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src) { return emu::warp_read(v, src, true); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int o) { return emu::warp_read(v, emu::t_lane ^ o, true); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, int d) { return emu::warp_read(v, emu::t_lane - d, emu::t_lane - d >= 0); }
static inline unsigned __ballot_sync(unsigned, bool pred)
{
    if (!emu::t_warp) return pred ? 1u : 0u;
    emu::t_warp->slot[emu::t_lane] = pred ? 1ull : 0ull;
    emu::t_warp->bar.wait();
    unsigned m = 0;
    for (int l = 0; l < 32; l++) m |= (unsigned)emu::t_warp->slot[l] << l;
    emu::t_warp->bar.wait();
    return m;
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }

// ---- bit casts, loads, math -----------------------------------------------------------------
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
static inline double __longlong_as_double(long long i) { double d; memcpy(&d, &i, 8); return d; }
static inline long long __double_as_longlong(double d) { long long i; memcpy(&i, &d, 8); return i; }
template <class T> static inline T __ldcs(const T *p) { return *p; }
#define __expf(x) expf(x)
// the three helpers that are inline PTX in the CUDA file (transform.py drops those bodies)
static inline float frcp(float x) { return 1.0f / x; }
static inline float frsqrt(float x) { return 1.0f / sqrtf(x); }
static inline void ld_256(const float4 *p, float4 &b, float4 &c) { b = p[0]; c = p[1]; }

// b200sph.cu replaces peer_now_ns (inline PTX, defined below) and the driver-API module
// loading under this macro
#define B200SPH_HOST_EMULATION 1
template <class T> static inline T __ldg(const T *p) { return *p; }
using std::isinf;
using std::max;
using std::min;

// ---- atomics (really atomic: kernels may run as concurrent threads) ---------------------------
static inline uint32_t atomicAdd(uint32_t *p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <class T> static inline T emu_atomic_minmax(T *p, T v, bool want_max)
{
    T o = __atomic_load_n(p, __ATOMIC_RELAXED);
    while ((want_max ? v > o : v < o) && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return o;
}
static inline unsigned atomicMax(unsigned *p, unsigned v) { return emu_atomic_minmax(p, v, true); }
static inline long long atomicMax(long long *p, long long v) { return emu_atomic_minmax(p, v, true); }
static inline long long atomicMin(long long *p, long long v) { return emu_atomic_minmax(p, v, false); }

// ---- runtime API ----------------------------------------------------------------------------------
typedef int cudaError_t;
#define cudaSuccess 0
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
struct cudaIpcMemHandle_t { char reserved[64]; };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
#define cudaStreamNonBlocking 1
#define cudaEventDisableTiming 2
#define cudaIpcMemLazyEnablePeerAccess 1
static inline const char *cudaGetErrorString(cudaError_t e) { return e ? "emulated CUDA error" : "no error"; }
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
// "device" memory: malloc for small blocks, anonymous mmap for >= 4 KiB so that a block can be
// turned into a shared mapping IN PLACE when another process asks for it (cudaIpc emulation,
// cuda_shim.cpp: memfd + /proc/<pid>/fd/<fd>) -- the slab decomposition's peer-memory halo
// then runs across the worker processes of the tests exactly as over NVLink
namespace emu {
int dev_alloc(void **p, size_t n);
int dev_free(void *p);
int ipc_export(void *handle64, void *p);
int ipc_import(void **p, const void *handle64);
int ipc_release(void *p);
}
static inline cudaError_t cudaMalloc(void **p, size_t n) { return emu::dev_alloc(p, n); }
static inline cudaError_t cudaMallocHost(void **p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFree(void *p) { return emu::dev_free(p); }
static inline cudaError_t cudaFreeHost(void *p) { return emu::dev_free(p); }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return 0; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return 0; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return 0; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return 0; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = (void *)0x10; return 0; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return 0; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = (void *)0x20; return 0; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (void *)0x20; return 0; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return 0; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return 0; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return 0; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 1e-3f; return 0; }  // nothing is timed here; non-zero so that rates stay finite
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { return emu::ipc_export(h->reserved, p); }
static inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { return emu::ipc_import(p, h.reserved); }
static inline cudaError_t cudaIpcCloseMemHandle(void *p) { return emu::ipc_release(p); }
// ---- what the peer protocol (b200sph_peer_*) needs: priorities and mapped pinned memory are
//      no-ops / plain memory here, fences are real (the ranks are concurrent OS processes) ----
#include <sched.h>
#include <time.h>
#define cudaHostAllocMapped 2
#define cudaErrorNotReady 600
static inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { return cudaMalloc(p, n); }
static inline cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return 0; }
static inline cudaError_t cudaDeviceGetStreamPriorityRange(int *lo, int *hi) { *lo = 0; *hi = -1; return 0; }
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned, int) { *s = (void *)0x11; return 0; }
static inline cudaError_t cudaStreamQuery(cudaStream_t) { return 0; }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __nanosleep(unsigned) { sched_yield(); }
template <class T> static inline T __ldcg(const T *p) { return *(const volatile T *)p; }
static inline unsigned long long peer_now_ns()
{
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (unsigned long long)ts.tv_sec * 1000000000ull + (unsigned long long)ts.tv_nsec;
}
