// simt_emu.h -- a small CPU emulator of the CUDA SIMT execution model, used to run the kernels of
// segmamba_b200/csrc/*.cu UNMODIFIED on the host for functional testing (bounds, indexing, barriers, parity with
// the oracle) when no GPU is at hand.
//
// TEST INFRASTRUCTURE ONLY.  Nothing in the product imports, links or falls back to this; the emulated library is
// built by tools/simt_emu/build.py into tools/simt_emu/_build/ and loaded only by tests/test_emu_*.py.  It says
// nothing about performance and does not model memory ordering: it checks what the code computes.
//
// Model
//   * every CUDA thread is a ucontext fiber; a thread block's fibers run on one OS thread, blocks of a grid are
//     distributed over OS threads (std::thread), so atomics are real atomics and __shared__ is per OS thread;
//   * a fiber runs until it reaches a collective (__syncthreads, __syncwarp, __shfl_*_sync, __ballot_sync, ...),
//     parks there, and is released when every live thread of the block / every live lane named by the mask has
//     arrived -- so convergence bugs deadlock loudly ("no runnable thread") instead of computing garbage;
//   * lanes are resumed in ascending or (SMB_EMU_REVERSE=1) descending order: a missing barrier between a
//     shared-memory write and a cross-lane read shows up as a wrong result in one of the two orders;
//   * shuffles from an exited lane or a lane outside the mask abort;
//   * cp.async copies are deferred until the issuing thread waits for their group, TMA bulk tensor copies until a thread waits
//     on the mbarrier they signal (box copy with the tensor map's swizzle and zero fill; the landed bytes must equal expect_tx),
//     so a missing wait / barrier reads NaN poison, and copies still in flight at thread exit abort;
//   * build.py --asan adds AddressSanitizer: out-of-bounds accesses of a kernel abort with the .cu source line.
#pragma once

#ifndef SMB_EMU
#error "simt_emu.h is only for the emulator build (-DSMB_EMU)"
#endif

#define __shared__ static thread_local
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#undef __launch_bounds__
#define __launch_bounds__(...)

#include <ucontext.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

// ---- built-in variables -------------------------------------------------------------------------
extern thread_local uint3 threadIdx, blockIdx;
extern thread_local dim3 blockDim, gridDim;
static constexpr int warpSize = 32;

namespace emu {

enum State : int { READY = 0, WAIT_WARP = 1, WAIT_BLOCK = 2, DONE = 3 };

struct Fiber {
    void *sp = nullptr;                // saved stack pointer (x86-64 switch) ...
    ucontext_t ctx;                    // ... or ucontext on other hosts
    State st = READY;
    unsigned wait_mask = 0;
    uint3 tid;
    int seq = 0;                       // number of warp collectives this lane has entered (double-buffer parity)
    unsigned last_part = 0;            // lanes that took part in this lane's most recent collective
    struct AsyncCopy { void *dst; const void *src; unsigned bytes; int group; };
    std::vector<AsyncCopy> async;      // cp.async copies issued but not yet waited for (performed at wait time, see below)
    int async_group = 0;               // index of the group currently being filled (cp.async.commit_group increments it)
};

struct Block {
    std::vector<Fiber> fibers;
    ucontext_t sched;
    void *sched_sp = nullptr;
    int cur = -1;
    int nthreads = 0;
    std::vector<uint64_t> xchg;        // [warp][parity][lane] exchange slots for shuffles / ballots
    std::vector<unsigned> part;        // [warp][parity] participants of the collective, recorded at release time
    unsigned char *dyn_smem = nullptr;
    const std::function<void()> *body = nullptr;
    struct PendingTma { void *dst; unsigned char map[128]; int coords[5]; int ncoords; uint64_t *bar; };
    std::vector<PendingTma> tma;       // bulk tensor copies issued, not yet performed
    struct BarState { uint64_t *bar; unsigned expected, arrived; int completed; };
    std::vector<BarState> bars;        // mbarrier bookkeeping, keyed by shared-memory address
};

extern thread_local Block *g_block;

[[noreturn]] void die(const char *msg);
void yield_wait(State st, unsigned mask);
void run_grid(const std::function<void()> &body, dim3 grid, dim3 block, size_t smem_bytes);
inline unsigned char *dyn_smem() { return g_block->dyn_smem; }

inline int lane_id() { return (int)((threadIdx.x + threadIdx.y * blockDim.x + threadIdx.z * blockDim.x * blockDim.y) & 31); }
inline int linear_tid() { return (int)(threadIdx.x + threadIdx.y * blockDim.x + threadIdx.z * blockDim.x * blockDim.y); }

// exchange one 64-bit payload across the lanes named by mask; returns the slot array of this collective
uint64_t *warp_exchange(unsigned mask, uint64_t mine);
bool lane_live_and_in_mask(int src_lane, unsigned mask);

template <typename T> inline uint64_t pack(T v) {
    static_assert(sizeof(T) <= 8, "shuffle payload too wide");
    uint64_t u = 0;
    std::memcpy(&u, &v, sizeof(T));
    return u;
}
template <typename T> inline T unpack(uint64_t u) {
    T v;
    std::memcpy(&v, &u, sizeof(T));
    return v;
}

template <typename K, typename... A> inline void launch(K kernel, dim3 grid, dim3 block, size_t smem, A... args) {
    std::function<void()> body = [=]() { kernel(args...); };
    run_grid(body, grid, block, smem);
}

}  // namespace emu

#define SMB_EMU_LAUNCH(kernel, grid, block, smem, ...) emu::launch(kernel, dim3(grid), dim3(block), (size_t)(smem), __VA_ARGS__)

// ---- synchronisation and warp collectives --------------------------------------------------------
inline void __syncthreads() { emu::yield_wait(emu::WAIT_BLOCK, 0); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_exchange(mask, 0); }

template <typename T> inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    const int lane = emu::lane_id();
    const int s = (lane & ~(width - 1)) | (src & (width - 1));
    uint64_t *slots = emu::warp_exchange(mask, emu::pack(v));
    if (!emu::lane_live_and_in_mask(s, mask)) emu::die("__shfl_sync reads a lane that exited or is outside the mask");
    return emu::unpack<T>(slots[s]);
}
template <typename T> inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    const int lane = emu::lane_id();
    const int s = lane ^ lanemask;
    uint64_t *slots = emu::warp_exchange(mask, emu::pack(v));
    if ((s & ~(width - 1)) != (lane & ~(width - 1))) return v;
    if (!emu::lane_live_and_in_mask(s, mask)) emu::die("__shfl_xor_sync reads a lane that exited or is outside the mask");
    return emu::unpack<T>(slots[s]);
}
template <typename T> inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const int lane = emu::lane_id();
    const int s = lane - (int)delta;
    uint64_t *slots = emu::warp_exchange(mask, emu::pack(v));
    if (s < (lane & ~(width - 1))) return v;
    if (!emu::lane_live_and_in_mask(s, mask)) emu::die("__shfl_up_sync reads a lane that exited or is outside the mask");
    return emu::unpack<T>(slots[s]);
}
template <typename T> inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    const int lane = emu::lane_id();
    const int s = lane + (int)delta;
    uint64_t *slots = emu::warp_exchange(mask, emu::pack(v));
    if (s > (lane | (width - 1))) return v;
    if (!emu::lane_live_and_in_mask(s, mask)) emu::die("__shfl_down_sync reads a lane that exited or is outside the mask");
    return emu::unpack<T>(slots[s]);
}
inline unsigned __ballot_sync(unsigned mask, int pred) {
    uint64_t *slots = emu::warp_exchange(mask, pred ? 1 : 0);
    unsigned r = 0;
    for (int l = 0; l < 32; ++l)
        if (((mask >> l) & 1) && emu::lane_live_and_in_mask(l, mask) && slots[l]) r |= 1u << l;
    return r;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) {
    uint64_t *slots = emu::warp_exchange(mask, pred ? 1 : 0);
    for (int l = 0; l < 32; ++l)
        if (((mask >> l) & 1) && emu::lane_live_and_in_mask(l, mask) && !slots[l]) return 0;
    return 1;
}
inline unsigned __activemask() { return 0xffffffffu; }

// ---- cp.async (LDGSTS).  The copy is DEFERRED until the issuing thread waits for its group: code that reads the destination
// without cp.async.wait_group / wait_all sees the NaN poison instead of data, and a thread that exits with copies in flight
// aborts -- the two ways such a pipeline goes wrong on hardware.  Visibility to other lanes still needs the barrier that the
// thread-order modes check.
namespace emu {
void cp_async_issue(void *smem_dst, const void *gmem_src, unsigned bytes);
void cp_async_commit();
void cp_async_wait(int allow_pending_groups);
}  // namespace emu

// ---- TMA (cp.async.bulk.tensor) + mbarrier.  A bulk tensor copy is queued on the block and performed -- box by box, with the
// tensor map's swizzle and zero fill of out-of-range coordinates -- when some thread waits on the mbarrier it signals; a wait
// whose phase can never complete (no copy queued, byte count different from expect_tx) aborts instead of spinning.
namespace emu {
void mbar_init(uint64_t *bar, int count);
void mbar_expect_tx(uint64_t *bar, unsigned bytes);
void mbar_wait(uint64_t *bar, unsigned parity);
void tma_load(void *smem_dst, const void *tensor_map, const int *coords, int ncoords, uint64_t *bar);
}  // namespace emu

// ---- atomics (blocks run on several OS threads) -----------------------------------------------------
inline float atomicAdd(float *addr, float val) {
    static_assert(sizeof(float) == sizeof(uint32_t), "");
    uint32_t *a = reinterpret_cast<uint32_t *>(addr);
    uint32_t old = __atomic_load_n(a, __ATOMIC_RELAXED), neu;
    float f;
    do {
        std::memcpy(&f, &old, 4);
        f += val;
        std::memcpy(&neu, &f, 4);
    } while (!__atomic_compare_exchange_n(a, &old, neu, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
    std::memcpy(&f, &old, 4);
    return f;
}
inline int atomicAdd(int *addr, int val) { return __atomic_fetch_add(addr, val, __ATOMIC_RELAXED); }
inline unsigned atomicAdd(unsigned *addr, unsigned val) { return __atomic_fetch_add(addr, val, __ATOMIC_RELAXED); }
inline unsigned long long atomicAdd(unsigned long long *addr, unsigned long long val) {
    return __atomic_fetch_add(addr, val, __ATOMIC_RELAXED);
}
inline int atomicMin(int *addr, int val) {
    int old = __atomic_load_n(addr, __ATOMIC_RELAXED);
    while (val < old && !__atomic_compare_exchange_n(addr, &old, val, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
inline unsigned atomicMax(unsigned *addr, unsigned val) {
    unsigned old = __atomic_load_n(addr, __ATOMIC_RELAXED);
    while (val > old && !__atomic_compare_exchange_n(addr, &old, val, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
inline unsigned long long atomicMax(unsigned long long *addr, unsigned long long val) {
    unsigned long long old = __atomic_load_n(addr, __ATOMIC_RELAXED);
    while (val > old && !__atomic_compare_exchange_n(addr, &old, val, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
// the lanes named by mask whose value equals this lane's
template <typename T> inline unsigned __match_any_sync(unsigned mask, T v) {
    uint64_t *slots = emu::warp_exchange(mask, emu::pack(v));
    unsigned r = 0;
    for (int l = 0; l < 32; ++l)
        if (((mask >> l) & 1) && emu::lane_live_and_in_mask(l, mask) && slots[l] == emu::pack(v)) r |= 1u << l;
    return r;
}
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __threadfence_block() { std::atomic_thread_fence(std::memory_order_seq_cst); }

// ---- math / bit-cast intrinsics ---------------------------------------------------------------------
inline float __expf(float x) { return std::exp(x); }
inline float __logf(float x) { return std::log(x); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __frcp_rn(float a) { return 1.f / a; }
inline float rsqrtf(float a) { return 1.f / std::sqrt(a); }
inline float __frsqrt_rn(float a) { return 1.f / std::sqrt(a); }
inline float __fmaf_rn(float a, float b, float c) { return std::fma(a, b, c); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline float exp2f_emu(float x) { return std::exp2(x); }
inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned i) { float f; std::memcpy(&f, &i, 4); return f; }
template <typename T> inline T __ldg(const T *p) { return *p; }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline long min(long a, long b) { return a < b ? a : b; }
inline long max(long a, long b) { return a > b ? a : b; }
inline float min(float a, float b) { return std::fmin(a, b); }
inline float max(float a, float b) { return std::fmax(a, b); }

// nvcc's cuda_runtime.h has a typed overload of cudaFuncSetAttribute for kernel symbols; the emulator has no limits to raise
template <class T> inline cudaError_t cudaFuncSetAttribute(T *, cudaFuncAttribute, int) { return cudaSuccess; }
