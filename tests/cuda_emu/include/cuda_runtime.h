// cuda_emu — TEST INFRASTRUCTURE ONLY.  A small CUDA-on-CPU emulation so the product's kernels and host code
// (live-video-magnification_b200/csrc/*.cu) can be compiled with g++ and their *logic* exercised by the parity
// tests in a container that has no GPU (tests/cuda_emu/build_emu.py -> tests/cuda_emu/libmagcore_emu.so).
// It is never shipped, never loaded by the product (lvm_b200.capi loads libmagcore_b200.so only; mc_create in
// that library still fails without an sm_90 device), and it says nothing about performance.
//
// Model: a kernel launch runs its CTAs one after another; the threads of a CTA are cooperative fibers
// (ucontext) scheduled round-robin by one OS thread, so __syncthreads / warp shuffles have their CUDA meaning,
// execution is deterministic, and AddressSanitizer sees every out-of-bounds or misaligned access a kernel makes.
// The device code paths are the real ones: the build defines __CUDACC__ and __CUDA_ARCH__=1000.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <tuple>
#include <utility>

#define MC_CUDA_EMU 1

// ---- qualifiers -------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))

#define __shared__ static
#define __constant__ static
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__

// ---- built-in vector types ---------------------------------------------------------------------------
struct uint3 { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    constexpr dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(8) float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(4) short2 { short x, y; };
struct alignas(8) short4 { short x, y, z, w; };
struct alignas(4) uchar4 { unsigned char x, y, z, w; };
struct alignas(2) uchar2 { unsigned char x, y; };
struct uchar3 { unsigned char x, y, z; };
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float3 make_float3(float x, float y, float z) { return {x, y, z}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
inline int2 make_int2(int x, int y) { return {x, y}; }
inline int4 make_int4(int x, int y, int z, int w) { return {x, y, z, w}; }
inline uint2 make_uint2(unsigned x, unsigned y) { return {x, y}; }
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return {x, y, z, w}; }
inline short2 make_short2(short x, short y) { return {x, y}; }
inline short4 make_short4(short x, short y, short z, short w) { return {x, y, z, w}; }
inline uchar4 make_uchar4(unsigned char x, unsigned char y, unsigned char z, unsigned char w) { return {x, y, z, w}; }
inline uchar2 make_uchar2(unsigned char x, unsigned char y) { return {x, y}; }

extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
constexpr int warpSize = 32;

// ---- fiber scheduler hooks (emu_runtime.cpp) ---------------------------------------------------------
namespace cuda_emu {
void launch(dim3 grid, dim3 block, size_t smem, void* stream, const char* name, const std::function<void()>& body);
void sync_threads();
unsigned shfl(unsigned value_bits, int src_lane_or_delta, int mode, int width);   // mode 0 idx, 1 up, 2 down, 3 xor
void yield_spin();   // a thread polling a flag another thread of the CTA will set
unsigned lane_id();
void* dyn_smem();    // the launch's dynamic shared memory (`extern __shared__`), 128-byte aligned
}  // namespace cuda_emu

typedef struct CUstream_st* cudaStream_t;
namespace cuda_emu {
// `k<<<grid, block, smem, stream>>>(args)` is rewritten by build_emu.py into
// `cuda_emu::Launcher(grid, block, smem, stream).run("k", (k), args)`.  The arguments are copied at the launch, as
// CUDA does; the work itself runs at once, or — with CUDA_EMU_ASYNC=1 — is queued on its stream and executed later in
// a random order that only respects stream order and event dependencies (see enqueue below).
void enqueue(void* stream, std::function<void()> work);
struct Launcher {
    dim3 grid, block;
    size_t smem;
    void* stream;
    Launcher(dim3 g, dim3 b, size_t sm = 0, cudaStream_t s = nullptr) : grid(g), block(b), smem(sm), stream(s) {}
    template <typename K, typename... A> void run(const char* name, K kernel, A&&... args) {
        auto packed = std::make_tuple(std::decay_t<A>(std::forward<A>(args))...);
        const dim3 g = grid, b = block;
        const size_t sm = smem;
        void* st = stream;
        enqueue(st, [=]() { launch(g, b, sm, st, name, [&]() { std::apply(kernel, packed); }); });
    }
};
}  // namespace cuda_emu

// ---- synchronisation / warp intrinsics ----------------------------------------------------------------
inline void __syncthreads() { cuda_emu::sync_threads(); }
inline void __syncwarp(unsigned = 0xffffffffu) { cuda_emu::shfl(0, 0, 0, 32); }   // a shuffle is a warp barrier
template <typename T> inline T emu_shfl_(T v, int arg, int mode, int width) {
    static_assert(sizeof(T) == 4, "32-bit shuffles only");
    unsigned b;
    std::memcpy(&b, &v, 4);
    b = cuda_emu::shfl(b, arg, mode, width);
    std::memcpy(&v, &b, 4);
    return v;
}
template <typename T> inline T __shfl_sync(unsigned, T v, int src, int width = 32) { return emu_shfl_(v, src, 0, width); }
template <typename T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int width = 32) { return emu_shfl_(v, (int)d, 1, width); }
template <typename T> inline T __shfl_down_sync(unsigned, T v, unsigned d, int width = 32) { return emu_shfl_(v, (int)d, 2, width); }
template <typename T> inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) { return emu_shfl_(v, m, 3, width); }

// ---- memory / math intrinsics --------------------------------------------------------------------------
template <typename T> inline T __ldg(const T* p) { return *p; }
inline int __float2int_rn(float x) {
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (-2147483647 - 1);
    return (int)std::nearbyintf(x);
}
inline float __saturatef(float x) { return x != x ? 0.0f : (x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x)); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return std::sqrt(a); }
inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
inline float __log2f(float x) { return std::log2(x); }
inline float __expf(float x) { return std::exp(x); }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline int __float_as_int(float f) { int u; std::memcpy(&u, &f, 4); return u; }
inline float __int_as_float(int u) { float f; std::memcpy(&f, &u, 4); return f; }
// dp2a.lo: c + (int16 lo of a) * (int8 byte 0 of b) + (int16 hi of a) * (int8 byte 1 of b)
inline int __dp2a_lo(int a, int b, int c) {
    return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)(b & 0xff) + (int)(int16_t)((unsigned)a >> 16) * (int)(int8_t)((b >> 8) & 0xff);
}
inline int __dp2a_hi(int a, int b, int c) {
    return c + (int)(int16_t)(a & 0xffff) * (int)(int8_t)((b >> 16) & 0xff) + (int)(int16_t)((unsigned)a >> 16) * (int)(int8_t)((b >> 24) & 0xff);
}
inline size_t __cvta_generic_to_shared(const void* p) { return reinterpret_cast<size_t>(p); }

inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline size_t min(size_t a, size_t b) { return a < b ? a : b; }
inline size_t max(size_t a, size_t b) { return a > b ? a : b; }
inline float min(float a, float b) { return std::fmin(a, b); }
inline float max(float a, float b) { return std::fmax(a, b); }

// single-OS-thread fibers: plain read-modify-write is atomic
inline unsigned atomicMin(unsigned* p, unsigned v) { unsigned o = *p; if (v < o) *p = v; return o; }
inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
inline int atomicMin(int* p, int v) { int o = *p; if (v < o) *p = v; return o; }
inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }
inline float atomicAdd(float* p, float v) { float o = *p; *p = o + v; return o; }

// ---- runtime API subset ------------------------------------------------------------------------------------
enum cudaError_t { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNoDevice = 100,
                   cudaErrorNotSupported = 801, cudaErrorUnknown = 999 };
typedef struct CUevent_st* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void* devicePointer; void* hostPointer; };
struct cudaDeviceProp {
    char name[256];
    size_t totalGlobalMem, sharedMemPerBlock, sharedMemPerBlockOptin;
    int major, minor, multiProcessorCount, warpSize, maxThreadsPerBlock, l2CacheSize;
};
enum cudaDriverEntryPointQueryResult { cudaDriverEntryPointSuccess = 0, cudaDriverEntryPointSymbolNotFound = 1, cudaDriverEntryPointVersionNotSufficent = 2 };
constexpr unsigned cudaStreamNonBlocking = 1, cudaStreamDefault = 0;
constexpr unsigned cudaEventDisableTiming = 2, cudaEventDefault = 0;
constexpr unsigned cudaHostAllocDefault = 0, cudaHostRegisterDefault = 0;
constexpr unsigned long long cudaEnableDefault = 0;

enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
template <typename F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int value) {
    return value <= 227 * 1024 ? cudaSuccess : cudaErrorInvalidValue;   // sm_90: at most 227 KB per CTA
}
const char* cudaGetErrorString(cudaError_t e);
cudaError_t cudaGetLastError();
cudaError_t cudaPeekAtLastError();
cudaError_t cudaGetDeviceCount(int* n);
cudaError_t cudaSetDevice(int d);
cudaError_t cudaGetDevice(int* d);
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int d);
cudaError_t cudaDeviceSynchronize();
cudaError_t cudaMalloc(void** p, size_t n);
cudaError_t cudaFree(void* p);
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned flags);
cudaError_t cudaMallocHost(void** p, size_t n);
cudaError_t cudaFreeHost(void* p);
cudaError_t cudaHostRegister(void* p, size_t n, unsigned flags);
cudaError_t cudaHostUnregister(void* p);
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p);
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k);
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t st = nullptr);
cudaError_t cudaMemcpy2D(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind k);
cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind k, cudaStream_t st = nullptr);
cudaError_t cudaMemset(void* d, int v, size_t n);
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st = nullptr);
cudaError_t cudaStreamCreate(cudaStream_t* s);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned flags);
cudaError_t cudaStreamDestroy(cudaStream_t s);
cudaError_t cudaStreamSynchronize(cudaStream_t s);
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned flags = 0);
cudaError_t cudaEventCreate(cudaEvent_t* e);
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags);
cudaError_t cudaEventDestroy(cudaEvent_t e);
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr);
cudaError_t cudaEventSynchronize(cudaEvent_t e);
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b);
cudaError_t cudaGetDriverEntryPoint(const char* symbol, void** fn, unsigned long long flags, cudaDriverEntryPointQueryResult* q = nullptr);
