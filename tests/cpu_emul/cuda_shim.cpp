// cuda_shim.cpp -- TEST INFRASTRUCTURE: the kernel launcher of the host emulation (cuda_shim.h)
//
// Lock-stepped lanes (WARP / BLOCK mode) are cooperative FIBERS on the calling OS thread
// (x86-64: a six-register stack switch; a barrier / shuffle / ballot that has to wait hands
// the core to the next lane), so a __syncthreads costs a few hundred nanoseconds instead of
// a round of kernel scheduling.  Elsewhere (or with B200SPH_EMUL_THREADS=1) every lane is a
// real OS thread, which is what this file did before and is kept as the cross-check: lanes
// then really run concurrently, atomics included.
#include "cuda_shim.h"

#include <cstdio>
#include <cstdlib>
#include <fcntl.h>
#include <map>
#include <memory>
#include <mutex>
#include <sys/mman.h>
#include <unistd.h>

namespace emu {
// ---- "device" allocations and the cudaIpc stand-in ------------------------------------------
struct Block { size_t size; int kind; int fd; };   // kind 0 malloc, 1 anonymous mmap, 2 shared (memfd), 3 imported
static std::map<void *, Block> g_blocks;
static std::mutex g_blocks_mu;
static size_t page_round(size_t n) { const size_t pg = (size_t)sysconf(_SC_PAGESIZE); return (n + pg - 1) / pg * pg; }

int dev_alloc(void **p, size_t n)
{
    if (n == 0) n = 1;
    Block b{n, 0, -1};
    if (n >= 4096) {
        b.size = page_round(n);
        b.kind = 1;
        *p = mmap(nullptr, b.size, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (*p == MAP_FAILED) { *p = nullptr; return 2; }
    } else {
        *p = malloc(n);
        if (!*p) return 2;
    }
    std::lock_guard<std::mutex> g(g_blocks_mu);
    g_blocks[*p] = b;
    return 0;
}

int dev_free(void *p)
{
    if (!p) return 0;
    Block b{0, 0, -1};
    {
        std::lock_guard<std::mutex> g(g_blocks_mu);
        auto it = g_blocks.find(p);
        if (it == g_blocks.end()) { free(p); return 0; }
        b = it->second;
        g_blocks.erase(it);
    }
    if (b.kind == 0) free(p);
    else munmap(p, b.size);
    if (b.fd >= 0) close(b.fd);
    return 0;
}

struct IpcHandle { int magic, pid, fd; unsigned long long size; };

// make the block a shared mapping of a memfd at the SAME address; the handle names the fd
int ipc_export(void *handle64, void *p)
{
    std::lock_guard<std::mutex> g(g_blocks_mu);
    auto it = g_blocks.find(p);
    if (it == g_blocks.end() || it->second.kind == 0 || it->second.kind == 3) return 3;
    Block &b = it->second;
    if (b.kind == 1) {
        const int fd = memfd_create("b200sph_emul_ipc", 0);
        if (fd < 0) return 3;
        if (ftruncate(fd, (off_t)b.size) != 0 || pwrite(fd, p, b.size, 0) != (ssize_t)b.size) { close(fd); return 3; }
        if (mmap(p, b.size, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_FIXED, fd, 0) != p) { close(fd); return 3; }
        b.kind = 2;
        b.fd = fd;
    }
    IpcHandle h{0x1bc, (int)getpid(), b.fd, (unsigned long long)b.size};
    memset(handle64, 0, 64);
    memcpy(handle64, &h, sizeof(h));
    return 0;
}

int ipc_import(void **p, const void *handle64)
{
    IpcHandle h;
    memcpy(&h, handle64, sizeof(h));
    if (h.magic != 0x1bc) return 3;
    char path[64];
    snprintf(path, sizeof(path), "/proc/%d/fd/%d", h.pid, h.fd);
    const int fd = open(path, O_RDWR);
    if (fd < 0) return 3;
    void *q = mmap(nullptr, (size_t)h.size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (q == MAP_FAILED) return 3;
    std::lock_guard<std::mutex> g(g_blocks_mu);
    g_blocks[q] = Block{(size_t)h.size, 3, -1};
    *p = q;
    return 0;
}

int ipc_release(void *p) { return dev_free(p); }

// the number of live "device" and pinned blocks (imported IPC mappings included): what a
// destroyed context must give back
extern "C" long long emu_live_blocks()
{
    std::lock_guard<std::mutex> g(g_blocks_mu);
    return (long long)g_blocks.size();
}

thread_local idx3 t_threadIdx, t_blockIdx, t_blockDim, t_gridDim;
thread_local WarpCtx *t_warp = nullptr;
thread_local BlockCtx *t_block = nullptr;
thread_local int t_lane = 0;

static void set_ids(long long grid, long long block, long long b, long long t)
{
    t_gridDim = idx3{(unsigned)grid, 1, 1};
    t_blockDim = idx3{(unsigned)block, 1, 1};
    t_blockIdx = idx3{(unsigned)b, 0, 0};
    t_threadIdx = idx3{(unsigned)t, 0, 0};
    t_lane = (int)(t & 31);
}

#if defined(__x86_64__)
#define EMU_FIBERS 1
extern "C" void emu_switch(void **save_sp, void *load_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size emu_switch,.-emu_switch
)");

struct Fiber {
    void *sp = nullptr;
    char *stack = nullptr;
    bool done = true;
    long long tid = 0;
    WarpCtx *warp = nullptr;
};
static const size_t FIBER_STACK = 512 * 1024;
struct FiberSet {
    std::vector<Fiber> f;
    void *main_sp = nullptr;
    int cur = -1;
    const std::function<void()> *body = nullptr;
    ~FiberSet() { for (auto &x : f) free(x.stack); }
};
static thread_local FiberSet *t_set = nullptr;

static void fiber_entry()
{
    FiberSet *S = t_set;
    Fiber &me = S->f[(size_t)S->cur];
    (*S->body)();
    me.done = true;
    emu_switch(&me.sp, S->main_sp);
    abort();   // a finished fiber is never resumed
}

static void run_fibers(long long grid, long long block, long long b, long long first, int n, BlockCtx *bc,
                       WarpCtx *wc, const std::function<void()> &body)
{
    static thread_local std::unique_ptr<FiberSet> pool;
    if (!pool) pool.reset(new FiberSet);
    FiberSet *S = pool.get();
    if ((int)S->f.size() < n) S->f.resize((size_t)n);
    S->body = &body;
    FiberSet *outer = t_set;
    t_set = S;
    for (int i = 0; i < n; i++) {
        Fiber &f = S->f[(size_t)i];
        if (!f.stack) f.stack = (char *)malloc(FIBER_STACK);
        uintptr_t top = ((uintptr_t)f.stack + FIBER_STACK) & ~(uintptr_t)15;
        void **sp = (void **)top;
        *--sp = nullptr;                 // keeps rsp = 8 (mod 16) at fiber_entry, as after a call
        *--sp = (void *)&fiber_entry;    // popped by emu_switch's ret
        for (int r = 0; r < 6; r++) *--sp = nullptr;
        f.sp = sp;
        f.done = false;
        f.tid = first + i;
        f.warp = bc ? &bc->warps[(size_t)(f.tid >> 5)] : wc;
    }
    int left = n;
    while (left > 0) {
        for (int i = 0; i < n; i++) {
            Fiber &f = S->f[(size_t)i];
            if (f.done) continue;
            S->cur = i;
            set_ids(grid, block, b, f.tid);
            t_block = bc;
            t_warp = f.warp;
            emu_switch(&S->main_sp, f.sp);
            if (f.done) left--;
        }
    }
    S->cur = -1;
    t_block = nullptr;
    t_warp = nullptr;
    t_set = outer;
}

void yield()
{
    FiberSet *S = t_set;
    if (S && S->cur >= 0) emu_switch(&S->f[(size_t)S->cur].sp, S->main_sp);
    else std::this_thread::yield();
}
#else
void yield() { std::this_thread::yield(); }
#endif

void launch(long long grid, long long block, int mode, const std::function<void()> &body)
{
#ifdef EMU_FIBERS
    static const bool use_threads = getenv("B200SPH_EMUL_THREADS") && atoi(getenv("B200SPH_EMUL_THREADS")) != 0;
#else
    static const bool use_threads = true;
#endif
    for (long long b = 0; b < grid; b++) {
        if (mode == SEQ) {
            for (long long t = 0; t < block; t++) {
                set_ids(grid, block, b, t);
                body();
            }
        } else if (mode == WARP) {   // warps are independent: one warp at a time, 32 lock-stepped lanes
            for (long long w = 0; w < (block + 31) / 32; w++) {
                WarpCtx wc;
#ifdef EMU_FIBERS
                if (!use_threads) {
                    run_fibers(grid, block, b, w * 32, 32, nullptr, &wc, body);   // block sizes are multiples of 32 in this library
                    continue;
                }
#endif
                std::vector<std::thread> lanes;
                for (int l = 0; l < 32; l++)
                    lanes.emplace_back([&, l] {
                        set_ids(grid, block, b, w * 32 + l);
                        t_warp = &wc;
                        if (w * 32 + l < block) body();
                        t_warp = nullptr;
                    });
                for (auto &t : lanes) t.join();
            }
        } else {                     // BLOCK: every thread of the block runs in lock step
            BlockCtx bc((int)block);
#ifdef EMU_FIBERS
            if (!use_threads) {
                run_fibers(grid, block, b, 0, (int)block, &bc, nullptr, body);
                continue;
            }
#endif
            std::vector<std::thread> ths;
            for (long long t = 0; t < block; t++)
                ths.emplace_back([&, t] {
                    set_ids(grid, block, b, t);
                    t_block = &bc;
                    t_warp = &bc.warps[(size_t)(t >> 5)];
                    body();
                    t_block = nullptr;
                    t_warp = nullptr;
                });
            for (auto &t : ths) t.join();
        }
    }
}
}  // namespace emu
