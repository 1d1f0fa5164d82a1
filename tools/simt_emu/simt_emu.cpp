// simt_emu.cpp -- scheduler of the CPU SIMT emulator (see simt_emu.h).  TEST INFRASTRUCTURE ONLY.
#include "simt_emu.h"

#include <memory>
#include <mutex>

thread_local uint3 threadIdx, blockIdx;
thread_local dim3 blockDim, gridDim;

// ---- context switch.  swapcontext() makes a sigprocmask system call per switch; on x86-64 a callee-saved-register switch
// in a few instructions is used instead (fibers never touch the signal mask, MXCSR or the x87 control word). ----
#if defined(__x86_64__)
#define SMB_EMU_FAST_SWITCH 1
extern "C" void smb_emu_switch(void **save_sp, void *load_sp);
asm(R"(
.text
.globl smb_emu_switch
.type smb_emu_switch,@function
smb_emu_switch:
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
.size smb_emu_switch,.-smb_emu_switch
)");
#endif

#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/common_interface_defs.h>
#define SMB_EMU_ASAN 1
#endif

namespace emu {

thread_local Block *g_block = nullptr;

// AddressSanitizer has to be told about every stack switch (build.py --asan: the memcheck mode of the emulator)
struct StackInfo { const void *bottom; size_t size; };
static thread_local StackInfo g_sched_stack = {nullptr, 0};

static inline void switch_stacks(void **save_sp, void *load_sp, const StackInfo *to, bool dying) {
#ifdef SMB_EMU_ASAN
    void *fake = nullptr;
    __sanitizer_start_switch_fiber(dying ? nullptr : &fake, to->bottom, to->size);
#endif
    smb_emu_switch(save_sp, load_sp);
#ifdef SMB_EMU_ASAN
    __sanitizer_finish_switch_fiber(fake, nullptr, nullptr);
#endif
}

static size_t stack_bytes() {
    static const size_t v = (getenv("SMB_EMU_STACK_KB") ? (size_t)atol(getenv("SMB_EMU_STACK_KB")) : 256) * 1024;
    return v;
}
// resume order of a block's threads: 0 ascending, 1 descending, >= 2 pseudo-random per scheduling round (value = seed)
static std::atomic<int> g_reverse{-1};
static int g_order_mode() {
    int v = g_reverse.load();
    if (v < 0) {
        v = getenv("SMB_EMU_REVERSE") ? atoi(getenv("SMB_EMU_REVERSE")) : 0;
        if (v < 0) v = 0;
        g_reverse.store(v);
    }
    return v;
}
static int worker_count() {
    static const int v = getenv("SMB_EMU_THREADS") ? atoi(getenv("SMB_EMU_THREADS")) : (int)std::thread::hardware_concurrency();
    return v > 0 ? v : 1;
}

[[noreturn]] void die(const char *msg) {
    fprintf(stderr, "simt_emu: %s (block %u,%u,%u thread %u,%u,%u)\n", msg, blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x,
            threadIdx.y, threadIdx.z);
    fflush(stderr);
    abort();
}

void yield_wait(State st, unsigned mask) {
    Block *b = g_block;
    Fiber &f = b->fibers[b->cur];
    f.st = st;
    f.wait_mask = mask;
#ifdef SMB_EMU_FAST_SWITCH
    switch_stacks(&f.sp, b->sched_sp, &g_sched_stack, false);
#else
    swapcontext(&f.ctx, &b->sched);
#endif
}

uint64_t *warp_exchange(unsigned mask, uint64_t mine) {
    Block *b = g_block;
    Fiber &f = b->fibers[b->cur];
    const int tid = linear_tid();
    const int warp = tid >> 5, lane = tid & 31;
    if (!((mask >> lane) & 1)) die("a lane calls a warp collective with a mask that does not name it");
    const int parity = f.seq & 1;
    uint64_t *slots = &b->xchg[(size_t)(warp * 2 + parity) * 32];
    slots[lane] = mine;
    f.seq++;
    yield_wait(WAIT_WARP, mask);
    f.last_part = b->part[(size_t)(warp * 2 + parity)];
    return slots;
}

bool lane_live_and_in_mask(int src_lane, unsigned mask) {
    Block *b = g_block;
    if (src_lane < 0 || src_lane > 31) return false;
    if (!((mask >> src_lane) & 1)) return false;
    return (b->fibers[b->cur].last_part >> src_lane) & 1;     // took part in the same collective (it may have exited since)
}

void cp_async_issue(void *smem_dst, const void *gmem_src, unsigned bytes) {
    Fiber &f = g_block->fibers[g_block->cur];
    if (bytes != 4 && bytes != 8 && bytes != 16) die("cp.async size must be 4, 8 or 16 bytes");
    if (((uintptr_t)smem_dst | (uintptr_t)gmem_src) & (bytes - 1)) die("cp.async source / destination not aligned to the copy size");
    f.async.push_back({smem_dst, gmem_src, bytes, f.async_group});
}
void cp_async_commit() { g_block->fibers[g_block->cur].async_group++; }
void cp_async_wait(int allow_pending_groups) {
    Fiber &f = g_block->fibers[g_block->cur];
    const int done_below = f.async_group - allow_pending_groups;      // groups with index < done_below must be complete
    size_t keep = 0;
    for (size_t i = 0; i < f.async.size(); ++i) {
        const Fiber::AsyncCopy &a = f.async[i];
        if (a.group < done_below) memcpy(a.dst, a.src, a.bytes);
        else f.async[keep++] = a;
    }
    f.async.resize(keep);
}

// ---- TMA + mbarrier model -----------------------------------------------------------------------------------------
struct TmapDescEmu {              // must match smb::TmapDesc (csrc/tma.cuh)
    const void *base;
    int rank, elem_bytes, swizzle64;
    uint64_t dims[5];
    uint64_t strides[5];
    uint32_t box[5];
};
static Block::BarState &bar_state(uint64_t *bar) {
    Block *b = g_block;
    for (auto &s : b->bars)
        if (s.bar == bar) return s;
    die("mbarrier used before mbarrier.init");
}
void mbar_init(uint64_t *bar, int count) {
    Block *b = g_block;
    if (count != 1) die("the emulator models single-arrival mbarriers only");
    for (auto &s : b->bars)
        if (s.bar == bar) { s = {bar, 0, 0, 0}; return; }
    b->bars.push_back({bar, 0, 0, 0});
}
void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    Block::BarState &s = bar_state(bar);
    if (s.expected) die("mbarrier.arrive.expect_tx on a phase that is already armed");
    s.expected = bytes;
}
void tma_load(void *smem_dst, const void *tensor_map, const int *coords, int ncoords, uint64_t *bar) {
    Block *b = g_block;
    Block::PendingTma p;
    p.dst = smem_dst;
    memcpy(p.map, tensor_map, 128);
    for (int i = 0; i < 5; ++i) p.coords[i] = i < ncoords ? coords[i] : 0;
    p.ncoords = ncoords;
    p.bar = bar;
    (void)bar_state(bar);
    if ((uintptr_t)((unsigned char *)smem_dst - b->dyn_smem) & 127) die("TMA destination must be 128-byte aligned in shared memory");
    b->tma.push_back(p);
}
static void tma_perform(Block *b, const Block::PendingTma &p, Block::BarState &s) {
    TmapDescEmu d;
    memcpy(&d, p.map, sizeof(d));
    if (d.rank != p.ncoords) die("TMA coordinate count differs from the tensor map's rank");
    const size_t inner_bytes = (size_t)d.box[0] * d.elem_bytes;
    size_t rows = 1;
    for (int i = 1; i < d.rank; ++i) rows *= d.box[i];
    const size_t dst_off0 = (size_t)((unsigned char *)p.dst - b->dyn_smem);
    if (d.swizzle64 && (inner_bytes != 64 || (dst_off0 & 511))) die("SWIZZLE_64B tile: 64-byte inner box and 512-byte aligned destination expected");
    for (size_t r = 0; r < rows; ++r) {
        size_t rem = r;                                          // box coordinates of this row in dims 1..rank-1
        bool inb = true;
        int64_t off = 0;
        for (int i = 1; i < d.rank; ++i) {
            const int64_t idx = (int64_t)p.coords[i] + (int64_t)(rem % d.box[i]);
            rem /= d.box[i];
            if (idx < 0 || idx >= (int64_t)d.dims[i]) inb = false;
            off += idx * (int64_t)d.strides[i - 1];
        }
        for (uint32_t e = 0; e < d.box[0]; ++e) {
            const int64_t i0 = (int64_t)p.coords[0] + e;
            size_t o = dst_off0 + r * inner_bytes + (size_t)e * d.elem_bytes;
            if (d.swizzle64) o ^= ((o >> 7) & 3) << 4;           // 16-byte chunk index ^= shared-address bits 7..8
            unsigned char *dst = b->dyn_smem + o;
            if (inb && i0 >= 0 && i0 < (int64_t)d.dims[0]) memcpy(dst, (const unsigned char *)d.base + off + i0 * d.elem_bytes, d.elem_bytes);
            else memset(dst, 0, d.elem_bytes);
        }
    }
    s.arrived += (unsigned)(rows * inner_bytes);
}
void mbar_wait(uint64_t *bar, unsigned parity) {
    Block *b = g_block;
    for (int spins = 0;; ++spins) {
        Block::BarState &s = bar_state(bar);
        if ((unsigned)(s.completed & 1) != parity) return;      // the phase with this parity has completed
        if (s.expected) {                                        // armed: the queued copies that signal it land now
            size_t keep = 0;
            for (size_t i = 0; i < b->tma.size(); ++i) {
                if (b->tma[i].bar == bar) tma_perform(b, b->tma[i], s);
                else b->tma[keep++] = b->tma[i];
            }
            b->tma.resize(keep);
            if (s.arrived > s.expected) die("more TMA bytes landed on an mbarrier than its expect_tx announced");
            if (s.arrived == s.expected) {
                s.completed++;
                s.expected = 0;
                s.arrived = 0;
                return;
            }
        }
        // not armed yet, or copies still to be issued by a thread that has not run: let the others run (try_wait spin)
        if (spins > 200000) die("mbarrier wait never completed (phase not armed, or fewer bytes issued than expect_tx)");
        yield_wait(READY, 0);
    }
}

static void fiber_entry() {
#ifdef SMB_EMU_ASAN
    {   // first time on this stack: complete the switch the scheduler started and learn the scheduler's stack bounds
        const void *bottom = nullptr;
        size_t size = 0;
        __sanitizer_finish_switch_fiber(nullptr, &bottom, &size);
        g_sched_stack = {bottom, size};
    }
#endif
    Block *b = g_block;
    (*b->body)();
    Fiber &f = b->fibers[b->cur];
    if (!f.async.empty()) die("thread exits with cp.async copies that were never waited for");
    if (!b->tma.empty()) {
        bool mine_last = true;
        for (const Fiber &o : b->fibers) mine_last = mine_last && (&o == &f || o.st == DONE);
        if (mine_last) die("block exits with TMA copies in flight that nobody waited for");
    }
    f.st = DONE;
#ifdef SMB_EMU_FAST_SWITCH
    switch_stacks(&f.sp, b->sched_sp, &g_sched_stack, true);     // never resumed
    abort();
#endif
    // ucontext: returning resumes uc_link (the scheduler)
}

static void run_block(Block &b, unsigned char *stacks) {
    const int n = b.nthreads;
    const size_t ss = stack_bytes();
    for (int i = 0; i < n; ++i) {
        Fiber &f = b.fibers[i];
        f.st = READY;
        f.seq = 0;
        f.wait_mask = 0;
        f.async.clear();
        f.async_group = 0;
        const unsigned x = i % blockDim.x, y = (i / blockDim.x) % blockDim.y, z = i / (blockDim.x * blockDim.y);
        f.tid = make_uint3(x, y, z);
#ifdef SMB_EMU_FAST_SWITCH
        // initial frame: six zeroed callee-saved registers, the entry point as return address, one pad word so that the
        // entry function sees the stack alignment of a normal call (rsp = 16n + 8)
        uintptr_t top = ((uintptr_t)(stacks + (size_t)(i + 1) * ss)) & ~(uintptr_t)15;
        void **sp = reinterpret_cast<void **>(top);
        *--sp = nullptr;
        *--sp = reinterpret_cast<void *>(&fiber_entry);
        for (int r = 0; r < 6; ++r) *--sp = nullptr;
        f.sp = sp;
#else
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = stacks + (size_t)i * ss;
        f.ctx.uc_stack.ss_size = ss;
        f.ctx.uc_link = &b.sched;
        makecontext(&f.ctx, fiber_entry, 0);
#endif
    }
    const int order = g_order_mode();
    const int nwarps = (n + 31) / 32;
    std::vector<int> perm(n);
    for (int i = 0; i < n; ++i) perm[i] = i;
    uint64_t rng = 0x9e3779b97f4a7c15ull ^ ((uint64_t)blockIdx.x * 0x100000001b3ull) ^ (uint64_t)order;
    for (;;) {
        bool ran = false;
        if (order >= 2) {                                   // a fresh pseudo-random resume order for every scheduling round
            for (int i = n - 1; i > 0; --i) {
                rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
                std::swap(perm[i], perm[(int)(rng % (uint64_t)(i + 1))]);
            }
        }
        for (int k = 0; k < n; ++k) {
            const int i = order >= 2 ? perm[k] : (order == 1 ? n - 1 - k : k);
            Fiber &f = b.fibers[i];
            if (f.st != READY) continue;
            b.cur = i;
            threadIdx = f.tid;
#ifdef SMB_EMU_FAST_SWITCH
            {
                const StackInfo fs = {stacks + (size_t)i * ss, ss};
                switch_stacks(&b.sched_sp, f.sp, &fs, false);
            }
#else
            swapcontext(&b.sched, &f.ctx);
#endif
            ran = true;
        }
        int live = 0, at_block = 0;
        for (int i = 0; i < n; ++i) {
            live += b.fibers[i].st != DONE;
            at_block += b.fibers[i].st == WAIT_BLOCK;
        }
        if (live == 0) return;
        bool released = false;
        if (at_block == live) {
            for (int i = 0; i < n; ++i)
                if (b.fibers[i].st == WAIT_BLOCK) b.fibers[i].st = READY;
            released = true;
        }
        for (int w = 0; w < nwarps; ++w) {
            const int lo = w * 32, hi = std::min(n, lo + 32);
            for (int i = lo; i < hi; ++i) {
                Fiber &f = b.fibers[i];
                if (f.st != WAIT_WARP) continue;
                bool ok = true;
                for (int j = lo; j < hi && ok; ++j) {
                    if (!((f.wait_mask >> (j - lo)) & 1)) continue;
                    const Fiber &g = b.fibers[j];
                    if (g.st == DONE) continue;                       // exited lanes are not waited for (as on hardware)
                    ok = g.st == WAIT_WARP && g.seq == f.seq && g.wait_mask == f.wait_mask;
                }
                if (!ok) continue;
                // release every lane of this collective together
                unsigned part = 0;
                const int parity = (f.seq - 1) & 1;
                for (int j = lo; j < hi; ++j) {
                    Fiber &g = b.fibers[j];
                    if (((f.wait_mask >> (j - lo)) & 1) && g.st == WAIT_WARP && g.seq == f.seq) {
                        g.st = READY;
                        part |= 1u << (j - lo);
                    }
                }
                b.part[(size_t)(w * 2 + parity)] = part;
                released = true;
            }
        }
        if (!ran && !released) {
            fprintf(stderr, "simt_emu: deadlock in block (%u,%u,%u): no runnable thread.  states:", blockIdx.x, blockIdx.y, blockIdx.z);
            for (int i = 0; i < n; ++i) fprintf(stderr, " %d:%d/%d", i, (int)b.fibers[i].st, b.fibers[i].seq);
            fprintf(stderr, "\n");
            abort();
        }
    }
}

void run_grid(const std::function<void()> &body, dim3 grid, dim3 block, size_t smem_bytes) {
    const long nblocks = (long)grid.x * grid.y * grid.z;
    const int nthreads = (int)(block.x * block.y * block.z);
    if (nblocks <= 0 || nthreads <= 0 || nthreads > 1024) {
        fprintf(stderr, "simt_emu: bad launch configuration grid=(%u,%u,%u) block=(%u,%u,%u)\n", grid.x, grid.y, grid.z, block.x, block.y,
                block.z);
        abort();
    }
    if (smem_bytes > 227 * 1024) {
        fprintf(stderr, "simt_emu: %zu bytes of dynamic shared memory exceed the 227 KB of an sm_90 CTA\n", smem_bytes);
        abort();
    }
    std::atomic<long> next{0};
    const int nw = (int)std::min<long>(worker_count(), nblocks);
    auto worker = [&]() {
        Block b;
        b.nthreads = nthreads;
        b.fibers.resize(nthreads);
        b.xchg.assign((size_t)((nthreads + 31) / 32) * 2 * 32, 0);
        b.part.assign((size_t)((nthreads + 31) / 32) * 2, 0);
        b.body = &body;
        std::unique_ptr<unsigned char[]> stacks(new unsigned char[(size_t)nthreads * stack_bytes()]);   // untouched pages cost nothing
        std::vector<unsigned char> smem(smem_bytes + 2048);
        b.dyn_smem = (unsigned char *)(((uintptr_t)smem.data() + 1023) & ~(uintptr_t)1023);     // CTA shared windows are 1 KB aligned
        g_block = &b;
        gridDim = grid;
        blockDim = block;
        for (;;) {
            const long id = next.fetch_add(1);
            if (id >= nblocks) break;
            blockIdx = make_uint3((unsigned)(id % grid.x), (unsigned)((id / grid.x) % grid.y), (unsigned)(id / ((long)grid.x * grid.y)));
            memset(b.dyn_smem, 0xff, smem_bytes);                       // NaN poison: shared memory is not zero on entry
            b.tma.clear();
            b.bars.clear();
            run_block(b, stacks.get());
        }
        g_block = nullptr;
    };
    if (nw == 1) {
        worker();
    } else {
        std::vector<std::thread> ts;
        for (int i = 0; i < nw; ++i) ts.emplace_back(worker);
        for (auto &t : ts) t.join();
    }
}

}  // namespace emu

// resume order of the threads of a block: 0 ascending, 1 descending, >= 2 pseudo-random (tests run several to expose
// missing barriers)
extern "C" __attribute__((visibility("default"))) void smb_emu_set_reverse(int mode) { emu::g_reverse.store(mode < 0 ? 0 : mode); }

// ---- the slice of the CUDA runtime the sources call: "device" memory is host memory, streams are synchronous ----
extern "C" {
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
cudaError_t cudaPeekAtLastError(void) { return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t) { return "simt_emu: no CUDA runtime"; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
cudaError_t cudaFuncSetAttribute(const void *, cudaFuncAttribute, int) { return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { memmove(d, s, n); return cudaSuccess; }
}
