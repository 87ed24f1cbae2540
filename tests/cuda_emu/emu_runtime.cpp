// cuda_emu — TEST INFRASTRUCTURE ONLY.  Runtime half of the CUDA-on-CPU emulation (see include/cuda_runtime.h):
// the fiber scheduler behind kernel launches, host-memory versions of the runtime API subset the product's host
// code uses, an emulated cuTensorMapEncodeTiled / bulk-tensor load, and a direct-DFT stand-in for cuFFT.
#include <cuda.h>
#include <cufft.h>
#include <ucontext.h>

#include <chrono>
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <vector>

#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/common_interface_defs.h>
#define EMU_ASAN 1
#endif

uint3 threadIdx{0, 0, 0}, blockIdx{0, 0, 0};
dim3 blockDim(1, 1, 1), gridDim(1, 1, 1);

namespace cuda_emu {
namespace {

enum State { READY, AT_BARRIER, AT_WARP, SPIN, DONE };
constexpr size_t kStack = 512 * 1024;

struct Fiber {
    ucontext_t ctx;
    char* stack = nullptr;
    State state = DONE;
    uint3 tid{0, 0, 0};
};
struct Warp {
    unsigned gen = 0;
    unsigned buf[2][32];
    unsigned stamp[2][32];   // generation + 1 in which the slot was written: a lane that has exited since still counts
};

ucontext_t g_sched;
std::vector<Fiber> g_fibers;
std::vector<Warp> g_warps;
int g_cur = -1;
const std::function<void()>* g_body = nullptr;
bool g_in_kernel = false;
unsigned long long g_launches = 0;

void switch_to(ucontext_t* from, ucontext_t* to, const void* to_stack, size_t to_size) {
#if defined(EMU_ASAN)
    void* fake = nullptr;
    __sanitizer_start_switch_fiber(&fake, to_stack, to_size);
    swapcontext(from, to);
    __sanitizer_finish_switch_fiber(fake, nullptr, nullptr);
#else
    (void)to_stack; (void)to_size;
    swapcontext(from, to);
#endif
}

const void* g_sched_stack = nullptr;
size_t g_sched_stack_size = 0;

void yield_to_scheduler() {
    Fiber& f = g_fibers[(size_t)g_cur];
    switch_to(&f.ctx, &g_sched, g_sched_stack, g_sched_stack_size);
    threadIdx = g_fibers[(size_t)g_cur].tid;
}

void fiber_entry() {
#if defined(EMU_ASAN)
    __sanitizer_finish_switch_fiber(nullptr, &g_sched_stack, &g_sched_stack_size);
#endif
    (*g_body)();
    g_fibers[(size_t)g_cur].state = DONE;
    Fiber& f = g_fibers[(size_t)g_cur];
#if defined(EMU_ASAN)
    __sanitizer_start_switch_fiber(nullptr, g_sched_stack, g_sched_stack_size);   // nullptr: this fiber is finished
#endif
    swapcontext(&f.ctx, &g_sched);
}

[[noreturn]] void die(const char* what, const char* name) {
    std::fprintf(stderr, "cuda_emu: %s in kernel %s, block (%u,%u,%u)\n", what, name, blockIdx.x, blockIdx.y, blockIdx.z);
    std::abort();
}

void run_block(unsigned n, const char* name) {
    const unsigned nwarps = (n + 31) / 32;
    g_warps.assign(nwarps, Warp{});
    for (auto& w : g_warps) std::memset(w.stamp, 0, sizeof(w.stamp));
    for (unsigned t = 0; t < n; ++t) {
        Fiber& f = g_fibers[t];
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = f.stack;
        f.ctx.uc_stack.ss_size = kStack;
        f.ctx.uc_link = &g_sched;
        makecontext(&f.ctx, fiber_entry, 0);
        f.state = READY;
        f.tid = uint3{t % blockDim.x, (t / blockDim.x) % blockDim.y, t / (blockDim.x * blockDim.y)};
    }
    // Poor man's racecheck: CUDA gives no order between the threads of a CTA except at barriers, so a kernel whose
    // result depends on the order in which the emulation runs them has a shared-memory (or global) race.
    // CUDA_EMU_ORDER=reverse | random runs the fibers in another order between synchronisation points.
    static const int order_mode = [] {
        const char* e = std::getenv("CUDA_EMU_ORDER");
        return !e ? 0 : (std::string(e) == "reverse" ? 1 : (std::string(e) == "random" ? 2 : 0));
    }();
    static unsigned long long lcg = 0x9E3779B97F4A7C15ull;
    static const char* only = std::getenv("CUDA_EMU_ORDER_KERNEL");   // restrict the permutation to kernels containing this
    const int mode = (only && !std::strstr(name, only)) ? 0 : order_mode;
    std::vector<unsigned> order(n);
    for (unsigned t = 0; t < n; ++t) order[t] = mode == 1 ? n - 1 - t : t;
    unsigned done = 0;
    while (done < n) {
        bool progress = false;
        if (mode == 2)
            for (unsigned i = n - 1; i > 0; --i) {
                lcg = lcg * 6364136223846793005ull + 1442695040888963407ull;
                std::swap(order[i], order[(unsigned)((lcg >> 33) % (i + 1))]);
            }
        for (unsigned oi = 0; oi < n; ++oi) {
            const unsigned t = order[oi];
            Fiber& f = g_fibers[t];
            if (f.state != READY && f.state != SPIN) continue;
            const bool was_spin = f.state == SPIN;
            f.state = READY;
            g_cur = (int)t;
            threadIdx = f.tid;
            switch_to(&g_sched, &f.ctx, f.stack, kStack);
            if (f.state == DONE) ++done;
            if (!(was_spin && f.state == SPIN)) progress = true;
        }
        // __syncthreads: every thread that has not exited must have arrived
        unsigned at_bar = 0;
        for (unsigned t = 0; t < n; ++t) at_bar += g_fibers[t].state == AT_BARRIER;
        if (at_bar && at_bar == n - done) {
            for (unsigned t = 0; t < n; ++t) if (g_fibers[t].state == AT_BARRIER) g_fibers[t].state = READY;
            progress = true;
        }
        // warp shuffles: every live lane of the warp must have arrived
        for (unsigned w = 0; w < nwarps; ++w) {
            unsigned live = 0, at = 0;
            for (unsigned t = w * 32; t < std::min(n, w * 32 + 32); ++t) {
                live += g_fibers[t].state != DONE;
                at += g_fibers[t].state == AT_WARP;
            }
            if (at && at == live) {
                g_warps[w].gen++;
                for (unsigned t = w * 32; t < std::min(n, w * 32 + 32); ++t) if (g_fibers[t].state == AT_WARP) g_fibers[t].state = READY;
                progress = true;
            }
        }
        if (!progress) die("deadlock (divergent __syncthreads / shuffle, or a flag nobody sets)", name);
    }
}

}  // namespace

namespace { void* g_dyn_smem = nullptr; }
void* dyn_smem() { return g_dyn_smem; }

void launch(dim3 grid, dim3 block, size_t smem, void*, const char* name, const std::function<void()>& body) {
    if (g_in_kernel) die("nested launch", name);
    if (smem > 227 * 1024) die("more than 227 KB of dynamic shared memory", name);
    g_dyn_smem = smem ? std::aligned_alloc(128, (smem + 127) / 128 * 128) : nullptr;   // fresh per launch: ASan sees overruns
    if (g_dyn_smem) std::memset(g_dyn_smem, 0xcd, smem);                               // shared memory starts as garbage
    const unsigned n = block.x * block.y * block.z;
    if (n == 0 || n > 1024) die("bad block size", name);
    if (grid.x == 0 || grid.y == 0 || grid.z == 0 || grid.y > 65535 || grid.z > 65535) die("bad grid size", name);
    if (g_fibers.size() < n) g_fibers.resize(n);
    for (unsigned t = 0; t < n; ++t)
        if (!g_fibers[t].stack) g_fibers[t].stack = static_cast<char*>(std::malloc(kStack));
    static const bool trace = std::getenv("CUDA_EMU_TRACE") != nullptr;
    if (trace) std::fprintf(stderr, "cuda_emu: launch %s grid (%u,%u,%u) block (%u,%u,%u)\n", name, grid.x, grid.y, grid.z, block.x, block.y, block.z);
    g_in_kernel = true;
    g_body = &body;
    gridDim = grid;
    blockDim = block;
    ++g_launches;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                blockIdx = uint3{bx, by, bz};
                run_block(n, name);
            }
    g_in_kernel = false;
    g_cur = -1;
    std::free(g_dyn_smem);
    g_dyn_smem = nullptr;
}

void sync_threads() {
    g_fibers[(size_t)g_cur].state = AT_BARRIER;
    yield_to_scheduler();
}

void yield_spin() {
    g_fibers[(size_t)g_cur].state = SPIN;
    yield_to_scheduler();
}

unsigned lane_id() { return (unsigned)g_cur & 31u; }

unsigned shfl(unsigned bits, int arg, int mode, int width) {
    const unsigned t = (unsigned)g_cur, lane = t & 31u;
    Warp& w = g_warps[t / 32];
    const unsigned mygen = w.gen;
    w.buf[mygen & 1][lane] = bits;
    w.stamp[mygen & 1][lane] = mygen + 1;
    g_fibers[t].state = AT_WARP;
    yield_to_scheduler();
    Warp& w2 = g_warps[t / 32];
    const int seg = (int)(lane & ~(unsigned)(width - 1));
    int src;
    switch (mode) {
    case 0: src = seg + (arg & (width - 1)); break;
    case 1: src = (int)lane - arg; if (src < seg) src = (int)lane; break;
    case 2: src = (int)lane + arg; if (src > seg + width - 1) src = (int)lane; break;
    default: src = (int)lane ^ arg; if (src > seg + width - 1 || src < seg) src = (int)lane; break;
    }
    // a source lane that did not take part in this shuffle (exited earlier, or beyond the block) yields the caller's own
    // value; one that took part and has exited SINCE is still a valid source
    if (w2.stamp[mygen & 1][src] != mygen + 1) return bits;
    return w2.buf[mygen & 1][src];
}

// ---- bulk tensor (TMA) ---------------------------------------------------------------------------------
void tma_load(void* dst, const CUtensorMap* tm, const int* c, uint64_t* bar) {
    // hardware requirements on the operands of cp.async.bulk.tensor: 128-byte aligned shared destination,
    // 64-byte aligned descriptor, 8-byte aligned mbarrier
    if ((reinterpret_cast<uintptr_t>(dst) & 127) || (reinterpret_cast<uintptr_t>(tm) & 63) || (reinterpret_cast<uintptr_t>(bar) & 7))
        die("misaligned TMA operand (shared destination 128 B, descriptor 64 B, mbarrier 8 B)", "bulk tensor load");
    const auto& m = tm->emu;
    const uint32_t rank = m.rank, es = m.elem_bytes;
    uint32_t box[5] = {1, 1, 1, 1, 1};
    for (uint32_t d = 0; d < rank; ++d) box[d] = m.box[d];
    unsigned char* out = static_cast<unsigned char*>(dst);
    for (uint32_t i4 = 0; i4 < box[4]; ++i4) for (uint32_t i3 = 0; i3 < box[3]; ++i3) for (uint32_t i2 = 0; i2 < box[2]; ++i2)
        for (uint32_t i1 = 0; i1 < box[1]; ++i1) for (uint32_t i0 = 0; i0 < box[0]; ++i0) {
            const uint32_t idx[5] = {i0, i1, i2, i3, i4};
            bool inb = true;
            size_t off = 0;
            for (uint32_t d = 0; d < rank; ++d) {
                const long long g = (long long)c[d] + idx[d];
                if (g < 0 || g >= (long long)m.dims[d]) { inb = false; break; }
                off += d == 0 ? (size_t)g * es : (size_t)g * m.strides[d - 1];
            }
            if (inb) std::memcpy(out, m.base + off, es); else std::memset(out, 0, es);
            out += es;
        }
    size_t bytes = es;
    for (uint32_t d = 0; d < rank; ++d) bytes *= box[d];
    mbar_complete_tx(bar, (unsigned)bytes);
}

namespace {
struct MbarState { unsigned arrivals_init = 1; long long pending_arrivals = 1, pending_tx = 0; };
std::map<const uint64_t*, MbarState> g_mbars;
void mbar_check(uint64_t* bar, MbarState& st) {
    if (st.pending_arrivals <= 0 && st.pending_tx == 0) {   // phase completes; the barrier re-arms for the next one
        *bar += 1;
        st.pending_arrivals = st.arrivals_init;
    }
}
}  // namespace

void mbar_init(uint64_t* bar, unsigned arrivals) {
    *bar = 0;
    g_mbars[bar] = MbarState{arrivals, (long long)arrivals, 0};
}
void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
    MbarState& st = g_mbars[bar];
    st.pending_tx += bytes;
    st.pending_arrivals -= 1;
    mbar_check(bar, st);
}
void mbar_complete_tx(uint64_t* bar, unsigned bytes) {
    MbarState& st = g_mbars[bar];
    st.pending_tx -= bytes;
    mbar_check(bar, st);
}

}  // namespace cuda_emu

// ---- emulated driver entry point ---------------------------------------------------------------------------
static CUresult emu_cuTensorMapEncodeTiled(CUtensorMap* tm, CUtensorMapDataType dt, cuuint32_t rank, void* base, const cuuint64_t* dims,
                                           const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr,
                                           CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
    // the constraints the real encoder enforces (CUDA driver API, cuTensorMapEncodeTiled)
    const uint32_t es = dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : dt == CU_TENSOR_MAP_DATA_TYPE_UINT16 ? 2 : 1;
    if (!tm || rank < 1 || rank > 5 || !base || (reinterpret_cast<uintptr_t>(base) & 15)) return CUDA_ERROR_INVALID_VALUE;
    for (cuuint32_t d = 0; d < rank; ++d) {
        if (dims[d] == 0 || dims[d] > (1ull << 32) || box[d] == 0 || box[d] > 256 || estr[d] == 0 || estr[d] > 8) return CUDA_ERROR_INVALID_VALUE;
        if (d + 1 < rank && ((strides[d] & 15) || strides[d] >= (1ull << 40))) return CUDA_ERROR_INVALID_VALUE;
    }
    if (((size_t)box[0] * es) & 15) return CUDA_ERROR_INVALID_VALUE;
    std::memset(tm, 0, sizeof(*tm));
    tm->emu.base = static_cast<const unsigned char*>(base);
    tm->emu.rank = rank;
    tm->emu.elem_bytes = es;
    for (cuuint32_t d = 0; d < rank; ++d) { tm->emu.dims[d] = dims[d]; tm->emu.box[d] = box[d]; if (d + 1 < rank) tm->emu.strides[d] = strides[d]; }
    return CUDA_SUCCESS;
}

// ---- streams and events --------------------------------------------------------------------------------------------
// Default: every operation runs at the call (one legal schedule).  CUDA_EMU_ASYNC=1: operations on a stream are queued
// and only executed when the host synchronises (stream / event / device sync, cudaFree), in a pseudo-random order
// (CUDA_EMU_SEED) that respects nothing but stream order and event waits — so a missing cudaStreamWaitEvent, a buffer
// reused before its consumer ran, or a host buffer touched while an async copy is pending shows up as a wrong result.
// As in CUDA, synchronous copies on the null stream do NOT wait for the (non-blocking) user streams.
namespace cuda_emu {
namespace {
struct EmuEvent {
    unsigned long long recorded = 0, completed = 0;   // sequence numbers of cudaEventRecord calls / executions
    std::chrono::steady_clock::time_point t;
};
struct Op {
    std::function<void()> work;       // kind 0
    int kind = 0;                     // 0 work, 1 record, 2 wait
    EmuEvent* ev = nullptr;
    unsigned long long seq = 0;
};
std::map<void*, std::deque<Op>> g_queues;
unsigned long long g_rng = 0;
bool async_mode() {
    static const bool on = [] {
        const char* e = std::getenv("CUDA_EMU_ASYNC");
        const char* sd = std::getenv("CUDA_EMU_SEED");
        g_rng = 0x2545F4914F6CDD1Dull ^ (sd ? std::strtoull(sd, nullptr, 10) * 0x9E3779B97F4A7C15ull : 0);
        return e && e[0] == '1';
    }();
    return on;
}
bool ready(const Op& op) { return op.kind != 2 || op.ev->completed >= op.seq; }
void execute(Op& op) {
    if (op.kind == 0) op.work();
    else if (op.kind == 1) { op.ev->completed = std::max(op.ev->completed, op.seq); op.ev->t = std::chrono::steady_clock::now(); }
}
// runs queued operations in a random legal order until done() holds
template <typename Pred> void drain_until(Pred done) {
    while (!done()) {
        std::vector<std::deque<Op>*> cand;
        for (auto& kv : g_queues)
            if (!kv.second.empty() && ready(kv.second.front())) cand.push_back(&kv.second);
        if (cand.empty()) {
            std::fprintf(stderr, "cuda_emu: stream deadlock — a wait on an event that is never recorded, or a synchronise on work that cannot run\n");
            std::abort();
        }
        g_rng = g_rng * 6364136223846793005ull + 1442695040888963407ull;
        std::deque<Op>* q = cand[(size_t)((g_rng >> 33) % cand.size())];
        Op op = std::move(q->front());
        q->pop_front();
        execute(op);
    }
}
void drain_all() {
    drain_until([] { for (auto& kv : g_queues) if (!kv.second.empty()) return false; return true; });
}
}  // namespace

void enqueue(void* stream, std::function<void()> work) {
    if (!async_mode() || stream == nullptr) { work(); return; }
    Op op;
    op.work = std::move(work);
    g_queues[stream].push_back(std::move(op));
}
}  // namespace cuda_emu

// ---- runtime API -----------------------------------------------------------------------------------------------
namespace {
std::map<const void*, std::pair<size_t, int>> g_allocs;   // ptr -> (bytes, 1 device / 2 pinned host / 3 registered)
using cuda_emu::EmuEvent;
}

const char* cudaGetErrorString(cudaError_t e) {
    switch (e) {
    case cudaSuccess: return "no error";
    case cudaErrorInvalidValue: return "invalid argument";
    case cudaErrorMemoryAllocation: return "out of memory";
    case cudaErrorNoDevice: return "no CUDA-capable device is detected";
    default: return "cuda_emu error";
    }
}
cudaError_t cudaGetLastError() { return cudaSuccess; }
cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : cudaErrorInvalidValue; }
cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int d) {
    if (d != 0) return cudaErrorInvalidValue;
    std::memset(p, 0, sizeof(*p));
    std::snprintf(p->name, sizeof(p->name), "cuda_emu (CPU fibers, not a GPU)");
    p->major = 9; p->minor = 0; p->multiProcessorCount = 132; p->warpSize = 32; p->maxThreadsPerBlock = 1024;
    p->totalGlobalMem = 8ull << 30; p->sharedMemPerBlock = 48 << 10; p->sharedMemPerBlockOptin = 227 << 10; p->l2CacheSize = 50 << 20;
    return cudaSuccess;
}
cudaError_t cudaDeviceSynchronize() { cuda_emu::drain_all(); return cudaSuccess; }
static cudaError_t emu_alloc(void** p, size_t n, int kind) {
    void* q = std::aligned_alloc(256, (n + 255) / 256 * 256 + 256);
    if (!q) return cudaErrorMemoryAllocation;
    std::memset(q, 0xcd, n);   // poison: kernels must not rely on zeroed allocations
    g_allocs[q] = {n, kind};
    *p = q;
    return cudaSuccess;
}
cudaError_t cudaMalloc(void** p, size_t n) { return emu_alloc(p, n, 1); }
cudaError_t cudaFree(void* p) {
    cuda_emu::drain_all();   // cudaFree synchronises the device
    if (p) { g_allocs.erase(p); std::free(p); }
    return cudaSuccess;
}
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return emu_alloc(p, n, 2); }
cudaError_t cudaMallocHost(void** p, size_t n) { return emu_alloc(p, n, 2); }
cudaError_t cudaFreeHost(void* p) { return cudaFree(p); }
cudaError_t cudaHostRegister(void* p, size_t n, unsigned) { g_allocs[p] = {n, 3}; return cudaSuccess; }
cudaError_t cudaHostUnregister(void* p) { g_allocs.erase(p); return cudaSuccess; }
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p) {
    std::memset(a, 0, sizeof(*a));
    a->type = cudaMemoryTypeUnregistered;
    auto it = g_allocs.upper_bound(p);
    if (it != g_allocs.begin()) {
        --it;
        const char* b = static_cast<const char*>(it->first);
        if (static_cast<const char*>(p) < b + it->second.first) a->type = it->second.second == 1 ? cudaMemoryTypeDevice : cudaMemoryTypeHost;
    }
    return cudaSuccess;
}
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) std::memmove(d, s, n); return cudaSuccess; }
// what kind of memory a pointer is: 1 device, 2 / 3 pinned host (allocated / registered), 0 pageable host
static int mem_kind(const void* p) {
    auto it = g_allocs.upper_bound(p);
    if (it == g_allocs.begin()) return 0;
    --it;
    return static_cast<const char*>(p) < static_cast<const char*>(it->first) + it->second.first ? it->second.second : 0;
}
// Asynchronous copies involving PAGEABLE host memory are not asynchronous in CUDA: a pageable source is staged before the
// call returns (so the caller may reuse or free it), and a copy into pageable memory returns only once it has completed.
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t st) {
    if (!n) return cudaSuccess;
    if (cuda_emu::async_mode() && st) {
        if (mem_kind(d) == 0) {                       // into pageable memory: synchronous with respect to the stream
            cudaStreamSynchronize(st);
            std::memmove(d, s, n);
            return cudaSuccess;
        }
        if (mem_kind(s) == 0) {                       // from pageable memory: staged now
            auto staged = std::make_shared<std::vector<unsigned char>>(static_cast<const unsigned char*>(s),
                                                                       static_cast<const unsigned char*>(s) + n);
            cuda_emu::enqueue(st, [=]() { std::memcpy(d, staged->data(), n); });
            return cudaSuccess;
        }
    }
    cuda_emu::enqueue(st, [=]() { std::memmove(d, s, n); });
    return cudaSuccess;
}
cudaError_t cudaMemcpy2D(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind) {
    if (w > dp || w > sp) return cudaErrorInvalidValue;
    for (size_t y = 0; y < h; ++y) std::memmove(static_cast<char*>(d) + y * dp, static_cast<const char*>(s) + y * sp, w);
    return cudaSuccess;
}
cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind k, cudaStream_t st) {
    if (w > dp || w > sp) return cudaErrorInvalidValue;
    if (cuda_emu::async_mode() && st && (mem_kind(d) == 0 || mem_kind(s) == 0)) {   // pageable side: see cudaMemcpyAsync
        cudaStreamSynchronize(st);
        return cudaMemcpy2D(d, dp, s, sp, w, h, k);
    }
    cuda_emu::enqueue(st, [=]() { cudaMemcpy2D(d, dp, s, sp, w, h, k); });
    return cudaSuccess;
}
cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) std::memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st) {
    cuda_emu::enqueue(st, [=]() { if (n) std::memset(d, v, n); });
    return cudaSuccess;
}
cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = reinterpret_cast<cudaStream_t>(new int(0)); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { return cudaStreamCreate(s); }
cudaError_t cudaStreamSynchronize(cudaStream_t s) {
    if (cuda_emu::async_mode() && s) cuda_emu::drain_until([s] { return cuda_emu::g_queues[s].empty(); });
    return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) {
    cudaStreamSynchronize(s);
    cuda_emu::g_queues.erase(s);
    delete reinterpret_cast<int*>(s);
    return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned) {
    auto* ev = reinterpret_cast<EmuEvent*>(e);
    if (!cuda_emu::async_mode() || !s || ev->recorded == 0) return cudaSuccess;   // never recorded: no-op, as in CUDA
    cuda_emu::Op op;
    op.kind = 2; op.ev = ev; op.seq = ev->recorded;                               // the latest record before this call
    cuda_emu::g_queues[s].push_back(std::move(op));
    return cudaSuccess;
}
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = reinterpret_cast<cudaEvent_t>(new EmuEvent{}); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
cudaError_t cudaEventDestroy(cudaEvent_t e) {
    if (cuda_emu::async_mode()) cuda_emu::drain_all();   // pending operations may still refer to it
    delete reinterpret_cast<EmuEvent*>(e);
    return cudaSuccess;
}
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) {
    auto* ev = reinterpret_cast<EmuEvent*>(e);
    const unsigned long long seq = ++ev->recorded;
    if (!cuda_emu::async_mode() || !s) { ev->completed = seq; ev->t = std::chrono::steady_clock::now(); return cudaSuccess; }
    cuda_emu::Op op;
    op.kind = 1; op.ev = ev; op.seq = seq;
    cuda_emu::g_queues[s].push_back(std::move(op));
    return cudaSuccess;
}
cudaError_t cudaEventSynchronize(cudaEvent_t e) {
    auto* ev = reinterpret_cast<EmuEvent*>(e);
    if (cuda_emu::async_mode()) cuda_emu::drain_until([ev] { return ev->completed >= ev->recorded; });
    return cudaSuccess;
}
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
    cudaEventSynchronize(a);
    cudaEventSynchronize(b);
    *ms = std::chrono::duration<float, std::milli>(reinterpret_cast<EmuEvent*>(b)->t - reinterpret_cast<EmuEvent*>(a)->t).count();
    return cudaSuccess;
}
cudaError_t cudaGetDriverEntryPoint(const char* symbol, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* q) {
    if (std::string(symbol) == "cuTensorMapEncodeTiled") {
        *fn = reinterpret_cast<void*>(&emu_cuTensorMapEncodeTiled);
        if (q) *q = cudaDriverEntryPointSuccess;
        return cudaSuccess;
    }
    *fn = nullptr;
    if (q) *q = cudaDriverEntryPointSymbolNotFound;
    return cudaSuccess;
}

// ---- cuFFT stand-in ------------------------------------------------------------------------------------------------
namespace {
struct Plan { int n, istride, idist, ostride, odist, batch; cufftType type; bool live; cudaStream_t stream; };
std::vector<Plan> g_plans(1);   // handle 0 is "no plan"
}
cufftResult cufftPlanMany(cufftHandle* plan, int rank, int* n, int*, int istride, int idist, int*, int ostride, int odist,
                          cufftType type, int batch) {
    if (rank != 1 || n[0] < 1 || batch < 1 || (type != CUFFT_R2C && type != CUFFT_C2R)) return CUFFT_INVALID_VALUE;
    g_plans.push_back(Plan{n[0], istride, idist, ostride, odist, batch, type, true, nullptr});
    *plan = (cufftHandle)g_plans.size() - 1;
    return CUFFT_SUCCESS;
}
cufftResult cufftCreate(cufftHandle* plan) {
    g_plans.push_back(Plan{0, 0, 0, 0, 0, 0, CUFFT_R2C, false, nullptr});
    *plan = (cufftHandle)g_plans.size() - 1;
    return CUFFT_SUCCESS;
}
cufftResult cufftSetAutoAllocation(cufftHandle p, int) { return (p <= 0 || (size_t)p >= g_plans.size()) ? CUFFT_INVALID_PLAN : CUFFT_SUCCESS; }
cufftResult cufftMakePlanMany(cufftHandle p, int rank, int* n, int*, int istride, int idist, int*, int ostride, int odist,
                              cufftType type, int batch, size_t* workSize) {
    if (p <= 0 || (size_t)p >= g_plans.size()) return CUFFT_INVALID_PLAN;
    if (rank != 1 || n[0] < 1 || batch < 1 || (type != CUFFT_R2C && type != CUFFT_C2R)) return CUFFT_INVALID_VALUE;
    g_plans[(size_t)p] = Plan{n[0], istride, idist, ostride, odist, batch, type, true, nullptr};
    if (workSize) *workSize = 256;   // a token amount, so the caller's shared-work-area path runs
    return CUFFT_SUCCESS;
}
cufftResult cufftSetWorkArea(cufftHandle p, void* w) {
    if (p <= 0 || (size_t)p >= g_plans.size()) return CUFFT_INVALID_PLAN;
    return w ? CUFFT_SUCCESS : CUFFT_INVALID_VALUE;
}
cufftResult cufftSetStream(cufftHandle p, cudaStream_t s) {
    if (p <= 0 || (size_t)p >= g_plans.size()) return CUFFT_INVALID_PLAN;
    g_plans[(size_t)p].stream = s;
    return CUFFT_SUCCESS;
}
cufftResult cufftDestroy(cufftHandle p) {
    if (p <= 0 || (size_t)p >= g_plans.size()) return CUFFT_INVALID_PLAN;
    if (cuda_emu::async_mode()) cuda_emu::drain_all();
    g_plans[(size_t)p].live = false;
    return CUFFT_SUCCESS;
}
static cufftResult exec_r2c(Plan p, cufftReal* in, cufftComplex* out);
static cufftResult exec_c2r(Plan p, cufftComplex* in, cufftReal* out);
cufftResult cufftExecR2C(cufftHandle h, cufftReal* in, cufftComplex* out) {
    if (h <= 0 || (size_t)h >= g_plans.size() || !g_plans[(size_t)h].live || g_plans[(size_t)h].type != CUFFT_R2C) return CUFFT_INVALID_PLAN;
    const Plan p = g_plans[(size_t)h];
    cuda_emu::enqueue(p.stream, [=]() { exec_r2c(p, in, out); });
    return CUFFT_SUCCESS;
}
cufftResult cufftExecC2R(cufftHandle h, cufftComplex* in, cufftReal* out) {
    if (h <= 0 || (size_t)h >= g_plans.size() || !g_plans[(size_t)h].live || g_plans[(size_t)h].type != CUFFT_C2R) return CUFFT_INVALID_PLAN;
    const Plan p = g_plans[(size_t)h];
    cuda_emu::enqueue(p.stream, [=]() { exec_c2r(p, in, out); });
    return CUFFT_SUCCESS;
}
static cufftResult exec_r2c(Plan p, cufftReal* in, cufftComplex* out) {
    const int n = p.n;
    std::vector<double> cs((size_t)n), sn((size_t)n), x((size_t)n);
    for (int j = 0; j < n; ++j) { cs[(size_t)j] = std::cos(2.0 * M_PI * j / n); sn[(size_t)j] = std::sin(2.0 * M_PI * j / n); }
    for (int b = 0; b < p.batch; ++b) {
        for (int j = 0; j < n; ++j) x[(size_t)j] = in[(size_t)b * p.idist + (size_t)j * p.istride];
        for (int k = 0; k <= n / 2; ++k) {
            double re = 0, im = 0;
            for (int j = 0; j < n; ++j) { const size_t t = (size_t)((long long)j * k % n); re += x[(size_t)j] * cs[t]; im -= x[(size_t)j] * sn[t]; }
            out[(size_t)b * p.odist + (size_t)k * p.ostride] = cufftComplex{(float)re, (float)im};
        }
    }
    return CUFFT_SUCCESS;
}
static cufftResult exec_c2r(Plan p, cufftComplex* in, cufftReal* out) {
    const int n = p.n;
    std::vector<double> cs((size_t)n), sn((size_t)n), re((size_t)n / 2 + 1), im((size_t)n / 2 + 1);
    for (int j = 0; j < n; ++j) { cs[(size_t)j] = std::cos(2.0 * M_PI * j / n); sn[(size_t)j] = std::sin(2.0 * M_PI * j / n); }
    for (int b = 0; b < p.batch; ++b) {
        for (int k = 0; k <= n / 2; ++k) {
            const cufftComplex c = in[(size_t)b * p.idist + (size_t)k * p.istride];
            re[(size_t)k] = c.x; im[(size_t)k] = c.y;
        }
        for (int j = 0; j < n; ++j) {
            double v = re[0];
            for (int k = 1; k <= n / 2; ++k) {
                const size_t t = (size_t)((long long)j * k % n);
                if (2 * k == n) v += re[(size_t)k] * cs[t];                       // Nyquist bin: real part only
                else v += 2.0 * (re[(size_t)k] * cs[t] - im[(size_t)k] * sn[t]);
            }
            out[(size_t)b * p.odist + (size_t)j * p.ostride] = (float)v;
        }
    }
    return CUFFT_SUCCESS;
}
