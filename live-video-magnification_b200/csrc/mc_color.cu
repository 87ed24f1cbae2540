// Color mode — device twin of magcore::magnifyColor (reference
// src/processing/magnification/MagnifyCore.hpp:163-206): Gaussian pyrDown chain, rolling temporal
// window kept as a device ring buffer, ideal band-pass along time with cuFFT (R2C -> CCS-mask
// multiply -> C2R), global min-max normalisation, pyrUp chain (+ bilinear resize), min-max stretch.
#include <cfloat>
#include <cmath>
#include <algorithm>
#include <cstring>

#include "mc_modes.h"

namespace mc {

namespace {

// monotonic float <-> uint encoding so atomicMin/atomicMax order like floats
__device__ __forceinline__ unsigned f2ord(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void k_mm_init(unsigned* mm, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) mm[i] = (i & 1) ? 0u : 0xffffffffu;  // even: min slot, odd: max slot
}

// u8 interleaved frame -> f32 planes [lanes*C][h][pitch], value = (float)u8  (MagnifyCore.hpp:168-169)
template <int C>
__global__ void k_u8_to_planes(const uint8_t* __restrict__ in, size_t step, size_t lane_stride, int w, int h,
                               float* __restrict__ out, int pitch, size_t plane) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, lane = blockIdx.z;
    if (x >= w) return;
    const uint8_t* p = in + (size_t)lane * lane_stride + (size_t)y * step + (size_t)x * C;
#pragma unroll
    for (int c = 0; c < C; ++c) out[(size_t)(lane * C + c) * plane + (size_t)y * pitch + x] = (float)__ldg(p + c);
}

// small pyramid level (pitched planes) -> one time slot of the ring, rows packed tight
__global__ void k_ring_append(const float* __restrict__ src, int w, int h, int pitch, size_t plane,
                              float* __restrict__ slot, int planes) {
    const size_t n = (size_t)planes * h * w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int pl = (int)(i / ((size_t)h * w));
        const int rem = (int)(i - (size_t)pl * h * w);
        const int y = rem / w, x = rem - y * w;
        slot[i] = src[(size_t)pl * plane + (size_t)y * pitch + x];
    }
}

// spectrum[k][i] *= mask[k]  (mulSpectrums with the CCS-packed 0/1 mask, TemporalFilter.cpp:45-48, SURVEY A.4).
// createIdealBandpassFilter (TemporalFilter.cpp:59-80) is a real 0/1 mask over the PACKED indices x (1 where
// fl <= x <= fh); mulSpectrums reads it back as the complex number m[2k-1] + i m[2k] per bin, real only for DC and
// Nyquist.  The mask is evaluated here from (fl, fh) — no host vector, no per-frame upload; `sc` carries DFT_SCALE of
// both transforms.
__global__ void k_mask_mul(float2* __restrict__ spec, size_t S, int nbins, int n, double fl, double fh, float sc) {
    const size_t total = S * nbins;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i / S);
        const int xr = k == 0 ? 0 : (2 * k == n ? n - 1 : 2 * k - 1);
        const bool has_im = k != 0 && 2 * k != n;
        const float2 m = make_float2(((double)xr >= fl && (double)xr <= fh) ? sc : 0.0f,
                                     (has_im && (double)(2 * k) >= fl && (double)(2 * k) <= fh) ? sc : 0.0f);
        const float2 v = spec[i];
        spec[i] = make_float2(v.x * m.x - v.y * m.y, v.x * m.y + v.y * m.x);
    }
}

// per-lane min/max over `nchunks` chunks of `chunk` contiguous floats (chunk t at base + t*chunk_stride + lane*chunk)
// Block-wide min/max -> one ordered-int atomic pair per CTA (a few hundred per launch instead of one per warp)
__device__ __forceinline__ void block_minmax_commit(float mn, float mx, unsigned* __restrict__ mm2) {
    __shared__ float s_mn[8], s_mx[8];
    for (int o = 16; o; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { mn = fminf(mn, s_mn[i]); mx = fmaxf(mx, s_mx[i]); }
        atomicMin(&mm2[0], f2ord(mn));
        atomicMax(&mm2[1], f2ord(mx));
    }
}

// min/max of one stream's part of the filtered window: nchunks contiguous runs of `chunk` floats, chunk_stride apart
// (TemporalFilter.cpp:55); 128-bit loads when the runs are 16-byte aligned
__global__ void __launch_bounds__(256) k_minmax(const float* __restrict__ base, size_t chunk, int nchunks, size_t chunk_stride,
                                                unsigned* __restrict__ mm, int vec_ok) {
    const int lane = blockIdx.y;
    float mn = INFINITY, mx = -INFINITY;
    for (int t = 0; t < nchunks; ++t) {
        const float* __restrict__ p = base + (size_t)t * chunk_stride + (size_t)lane * chunk;
        if (vec_ok) {
            const float4* __restrict__ p4 = reinterpret_cast<const float4*>(p);
            for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < chunk / 4; i += (size_t)gridDim.x * blockDim.x) {
                const float4 v = __ldg(p4 + i);
                mn = fminf(fminf(mn, fminf(v.x, v.y)), fminf(v.z, v.w));
                mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
            }
        } else {
            for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < chunk; i += (size_t)gridDim.x * blockDim.x) {
                const float v = __ldg(p + i);
                mn = fminf(mn, v);
                mx = fmaxf(mx, v);
            }
        }
    }
    block_minmax_commit(mn, mx, mm + 2 * lane);
}

__global__ void k_select(const float* __restrict__ col, const unsigned* __restrict__ mm, int C, int w, int h,
                         float alpha, float* __restrict__ dst, int pitch, size_t plane, int planes) {
    const size_t n = (size_t)planes * h * w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int pl = (int)(i / ((size_t)h * w));
        const int rem = (int)(i - (size_t)pl * h * w);
        const int y = rem / w, x = rem - y * w;
        const int lane = pl / C;
        const double smin = (double)ord2f(mm[2 * lane]), smax = (double)ord2f(mm[2 * lane + 1]);
        const double scale = (smax - smin > DBL_EPSILON) ? 1.0 / (smax - smin) : 0.0;   // cv::normalize NORM_MINMAX
        const double shift = 0.0 - smin * scale;
        const float v = fmaf(col[i], (float)scale, (float)shift);
        dst[(size_t)pl * plane + (size_t)y * pitch + x] = v * alpha;
    }
}

// cv::pyrUp with the default destination size 2w x 2h (SpatialFilter.cpp:45)
__global__ void __launch_bounds__(256) k_pyrup2x(Level ls, Level ld, const float* __restrict__ src,
                                                 float* __restrict__ dst) {
    // tile = 64 x 32 destination pixels, thread = 4 x 2 block: the 34 x 18 source window (pyrUp's border rule applied to
    // the indices) goes to shared memory once, the row pass and the column pass run in registers, 128-bit stores
    __shared__ __align__(16) float sD[18][36];
    const int plane = blockIdx.z;
    const int x0 = blockIdx.x * 64, y0 = blockIdx.y * 32;
    const float* __restrict__ s = src + (size_t)plane * ls.plane;
    for (int idx = threadIdx.x; idx < 18 * 34; idx += 256) {
        const int k = idx / 34, j = idx - k * 34;
        const int iy = upsrc(y0 / 2 - 1 + k, ls.h), ix = upsrc(x0 / 2 - 1 + j, ls.w);
        sD[k][j] = __ldg(s + (size_t)iy * ls.pitch + ix);
    }
    __syncthreads();
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int gx = x0 + 4 * tx;
    if (gx >= ld.w) return;
    float e[3][4];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float2 p0 = *reinterpret_cast<const float2*>(&sD[ty + q][2 * tx]);
        const float2 p1 = *reinterpret_cast<const float2*>(&sD[ty + q][2 * tx + 2]);
        e[q][0] = __fadd_rn(__fmaf_rn(p0.y, 6.0f, p0.x), p1.x);
        e[q][1] = __fmul_rn(__fadd_rn(p0.y, p1.x), 4.0f);
        e[q][2] = __fadd_rn(__fmaf_rn(p1.x, 6.0f, p0.y), p1.y);
        e[q][3] = __fmul_rn(__fadd_rn(p1.x, p1.y), 4.0f);
    }
    float* __restrict__ d = dst + (size_t)plane * ld.plane;
#pragma unroll
    for (int ry = 0; ry < 2; ++ry) {
        const int gy = y0 + 2 * ty + ry;
        if (gy >= ld.h) continue;
        float o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
            o[i] = ry ? __fmul_rn(__fmul_rn(__fadd_rn(e[1][i], e[2][i]), 4.0f), 1.0f / 64.0f)
                      : __fmul_rn(__fadd_rn(__fmaf_rn(e[1][i], 6.0f, e[0][i]), e[2][i]), 1.0f / 64.0f);
        // rows are padded to a multiple of 32 floats, so a full float4 at gx < w is always in-bounds
        *reinterpret_cast<float4*>(d + (size_t)gy * ld.pitch + gx) = make_float4(o[0], o[1], o[2], o[3]);
    }
}


// cv::resize(INTER_LINEAR) on f32 planes (SpatialFilter.cpp:48): horizontal then vertical lerp
__global__ void k_resize_linear(Level ls, Level ld, const float* __restrict__ src, float* __restrict__ dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, plane = blockIdx.z;
    if (x >= ld.w) return;
    const double sx_scale = (double)ls.w / ld.w, sy_scale = (double)ls.h / ld.h;
    float fx = (float)((x + 0.5) * sx_scale - 0.5);
    int sx = (int)floorf(fx);
    fx -= sx;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= ls.w - 1) { fx = 0.f; sx = ls.w - 1; }
    float fy = (float)((y + 0.5) * sy_scale - 0.5);
    int sy = (int)floorf(fy);
    fy -= sy;
    if (sy < 0) { fy = 0.f; sy = 0; }
    if (sy >= ls.h - 1) { fy = 0.f; sy = ls.h - 1; }
    const int sx1 = min(sx + 1, ls.w - 1), sy1 = min(sy + 1, ls.h - 1);
    const float* s = src + (size_t)plane * ls.plane;
    const float r0 = s[(size_t)sy * ls.pitch + sx] * (1.f - fx) + s[(size_t)sy * ls.pitch + sx1] * fx;
    const float r1 = s[(size_t)sy1 * ls.pitch + sx] * (1.f - fx) + s[(size_t)sy1 * ls.pitch + sx1] * fx;
    dst[(size_t)plane * ld.plane + (size_t)y * ld.pitch + x] = r0 * (1.f - fy) + r1 * fy;
}

// min/max of output = input + colorImg per lane (MagnifyCore.hpp:197-201)
__global__ void __launch_bounds__(256) k_sum_minmax(const float* __restrict__ a, const float* __restrict__ b, Level l, int C,
                                                    unsigned* __restrict__ mm) {
    // one stream per blockIdx.y; the CTAs of a stream share its C * h rows, each row read as 128-bit vectors
    const int lane = blockIdx.y;
    float mn = INFINITY, mx = -INFINITY;
    const int rows = C * l.h, w4 = l.w >> 2;
    for (int r = blockIdx.x; r < rows; r += gridDim.x) {
        const int c = r / l.h, y = r - c * l.h;
        const size_t o = (size_t)(lane * C + c) * l.plane + (size_t)y * l.pitch;
        const float4* __restrict__ a4 = reinterpret_cast<const float4*>(a + o);
        const float4* __restrict__ b4 = reinterpret_cast<const float4*>(b + o);
        for (int i = threadIdx.x; i < w4; i += 256) {
            const float4 u = __ldg(a4 + i), v = __ldg(b4 + i);
            const float s0 = u.x + v.x, s1 = u.y + v.y, s2 = u.z + v.z, s3 = u.w + v.w;
            mn = fminf(fminf(mn, fminf(s0, s1)), fminf(s2, s3));
            mx = fmaxf(fmaxf(mx, fmaxf(s0, s1)), fmaxf(s2, s3));
        }
        for (int x = 4 * w4 + threadIdx.x; x < l.w; x += 256) {
            const float sv = __ldg(a + o + x) + __ldg(b + o + x);
            mn = fminf(mn, sv);
            mx = fmaxf(mx, sv);
        }
    }
    block_minmax_commit(mn, mx, mm + 2 * lane);
}


// out8u = convertTo(input + colorImg, 255/(max-min), -min*255/(max-min))  (MagnifyCore.hpp:202-203)
template <int C>
__global__ void k_color_egress(const float* __restrict__ a, const float* __restrict__ b, Level l,
                               const unsigned* __restrict__ mm, uint8_t* __restrict__ out, size_t step,
                               size_t lane_stride, float* __restrict__ fout) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, lane = blockIdx.z;
    if (x >= l.w) return;
    const double mn = (double)ord2f(mm[2 * lane]), mx = (double)ord2f(mm[2 * lane + 1]);
    const float sa = (float)(255.0 / (mx - mn)), sb = (float)(-mn * 255.0 / (mx - mn));
    uint8_t* q = out + (size_t)lane * lane_stride + (size_t)y * step + (size_t)x * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const size_t o = (size_t)(lane * C + c) * l.plane + (size_t)y * l.pitch + x;
        const float v = a[o] + b[o];
        q[c] = scaled_to_u8(v, sa, sb);
        if (fout) fout[(((size_t)lane * l.h + y) * l.w + x) * C + c] = v;
    }
}

inline unsigned cdiv(int a, int b) { return (unsigned)((a + b - 1) / b); }
inline unsigned gs_blocks(size_t n) {
    size_t b = (n + 255) / 256;
    return (unsigned)(b < 1 ? 1 : (b > 132 * 16 ? 132 * 16 : b));
}

}  // namespace

void ColorMode::reset() {
    for (auto& kv : plans) {
        if (kv.second.r2c) cufftDestroy(kv.second.r2c);
        if (kv.second.c2r) cufftDestroy(kv.second.c2r);
    }
    plans.clear();
    plan_signals = 0;
    fft_work = nullptr;      // owned by the arena
    fft_work_bytes = 0;
    arena.release();
    lv.clear(); G.clear(); U.clear(); ulv.clear();
    ring = work = nullptr; spec = nullptr; minmax = nullptr;
    allocated = false;
    count = head = 0;
    ring_cap = ring_mod = 0;
}

#define CUFFT_CK(call)                                                            \
    do {                                                                          \
        cufftResult r__ = (call);                                                 \
        if (r__ != CUFFT_SUCCESS) {                                               \
            *ctx.err = std::string(#call) + ": cufft error " + std::to_string((int)r__); \
            return MC_ERR_CUDA;                                                   \
        }                                                                         \
    } while (0)

mc_status ColorMode::process(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int nlevels, int* produced) {
    *produced = 0;
    const int want_cap = optimal_buffer_size((int)p.framerate);  // MagnifyCore.hpp:176
    const int C = io.channels;
    const int planes = lanes * C;
    if (!allocated) {
        reset();
        levels = nlevels; channels = C; w = io.w; h = io.h;
        lv.resize((size_t)levels + 1);
        int cw = w, ch = h;
        for (int l = 0; l <= levels; ++l) {
            lv[(size_t)l] = make_level(cw, ch);
            cw = (cw + 1) / 2; ch = (ch + 1) / 2;
        }
        G.assign((size_t)levels + 1, nullptr);
        for (int l = 0; l <= levels; ++l) MCK(arena.alloc(&G[(size_t)l], (size_t)planes * lv[(size_t)l].plane));
        const Level& ls = lv[(size_t)levels];
        small_rows = ls.w * ls.h;
        ulv.resize((size_t)levels + 1);
        U.assign((size_t)levels + 2, nullptr);
        int uw = ls.w, uh = ls.h;
        for (int i = 0; i <= levels; ++i) {
            ulv[(size_t)i] = make_level(uw, uh);
            MCK(arena.alloc(&U[(size_t)i], (size_t)planes * ulv[(size_t)i].plane));
            uw *= 2; uh *= 2;
        }
        if (ulv[(size_t)levels].w != w || ulv[(size_t)levels].h != h)
            MCK(arena.alloc(&U[(size_t)levels + 1], (size_t)planes * lv[0].plane));
        void* mmv = nullptr;
        MCK(arena.alloc_bytes(&mmv, sizeof(unsigned) * 4 * (size_t)lanes));
        minmax = (float*)mmv;
        allocated = true;
    }
    const size_t S = (size_t)planes * small_rows;  // signals (pixels x channels x lanes)
    // Ring geometry.  `ring_mod` is the LOGICAL ring size (slots are taken modulo it), `ring_cap` the allocation.  It
    // follows the window cap the frame rate asks for; when that changes (rare: a UI action) the window is laid out
    // once in logical order — into a bigger allocation when needed, the replaced buffers being freed — so that the
    // invariant "head == 0 or count == ring_mod" holds from then on and no per-frame compaction is ever needed.  A
    // window that is longer than a lowered cap keeps its length, as the reference's does (it drops one column per
    // appended column, SpatialFilter.cpp:73-83).
    const int want_mod = std::max(std::max(want_cap, count), 2);
    if (ring == nullptr || want_mod != ring_mod) {
        if (ring_cap < want_mod || ring == nullptr) {
            float *nring = nullptr, *nwork = nullptr;
            void* nspec = nullptr;
            MCK(arena.alloc(&nring, (size_t)want_mod * S));
            MCK(arena.alloc(&nwork, (size_t)want_mod * S));
            MCK(arena.alloc_bytes(&nspec, sizeof(cufftComplex) * (size_t)(want_mod / 2 + 1) * S));
            for (int t = 0; t < count; ++t)
                MCK(cudaMemcpyAsync(nring + (size_t)t * S, ring + (size_t)((head + t) % ring_mod) * S, S * sizeof(float),
                                    cudaMemcpyDeviceToDevice, ctx.stream));
            if (ring) {   // cudaFree orders itself after the copies above (it synchronises the device)
                arena.free_block(ring); arena.free_block(work); arena.free_block(spec);
            }
            ring = nring; work = nwork; spec = (cufftComplex*)nspec;
            ring_cap = want_mod;
        } else if (head != 0) {
            for (int t = 0; t < count; ++t)
                MCK(cudaMemcpyAsync(work + (size_t)t * S, ring + (size_t)((head + t) % ring_mod) * S, S * sizeof(float),
                                    cudaMemcpyDeviceToDevice, ctx.stream));
            std::swap(ring, work);
        }
        head = 0;
        ring_mod = want_mod;
    }

    // ingest + Gaussian chain (SpatialFilter.cpp:13-23)
    {
        dim3 grid(cdiv(w, 256), h, lanes);
        if (C == 3) { const bool pp = ctx.prof && ctx.prof->begin("u8_to_planes", 0, ctx.stream); k_u8_to_planes<3><<<grid, 256, 0, ctx.stream>>>(io.in, io.in_step, io.in_lane_stride, w, h, G[0], lv[0].pitch, lv[0].plane); if (pp) ctx.prof->end(ctx.stream); }
        else { const bool pp = ctx.prof && ctx.prof->begin("u8_to_planes", 0, ctx.stream); k_u8_to_planes<1><<<grid, 256, 0, ctx.stream>>>(io.in, io.in_step, io.in_lane_stride, w, h, G[0], lv[0].pitch, lv[0].plane); if (pp) ctx.prof->end(ctx.stream); }
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    for (int l = 0; l < levels; ++l) {
        LevelArgs a;
        a.in_kind = 0; a.g = G[(size_t)l]; a.in_plane = lv[(size_t)l].plane; a.in_row = lv[(size_t)l].pitch;
        a.channels = C; a.lf = lv[(size_t)l]; a.lc = lv[(size_t)l + 1]; a.g_next = G[(size_t)l + 1];
        a.planes = planes; a.band = 0;
        LAUNCH("gauss_down", l, launch_down(a, ctx.stream));
    }
    // append to the rolling window; once full drop the oldest column (SpatialFilter.cpp:63-84)
    const Level& ls = lv[(size_t)levels];
    {
        const int slot = (head + count) % ring_mod;
        const bool pp = ctx.prof && ctx.prof->begin("ring_append", 0, ctx.stream);
        k_ring_append<<<gs_blocks(S), 256, 0, ctx.stream>>>(G[(size_t)levels], ls.w, ls.h, ls.pitch, ls.plane, ring + (size_t)slot * S, planes);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
        ++count;
        if (count > want_cap && want_cap > 0) {
            head = (head + 1) % ring_mod;
            --count;
        }
    }
    if (count < 2) return MC_OK;  // MagnifyCore.hpp:180 (passthrough)
    const int n = count;

    // ideal temporal band-pass (TemporalFilter.cpp:24-57) on the physical column order.  The DFT length is the current
    // window length (2 ... cap, every value once during warm-up): plans are cached per length and share one work area
    // (they run one after another on the handle's stream), so warm-up costs one plan build per length per stream
    // geometry instead of two cufftPlanMany + workspace malloc/free per frame.
    if (plan_signals != S) {
        for (auto& kv : plans) { cufftDestroy(kv.second.r2c); cufftDestroy(kv.second.c2r); }
        plans.clear();
        plan_signals = S;
    }
    auto it = plans.find(n);
    if (it == plans.end()) {
        FftPlans pl;
        int nn[1] = {n};
        int inembed[1] = {n}, onembed[1] = {n / 2 + 1};
        size_t ws_a = 0, ws_b = 0;
        CUFFT_CK(cufftCreate(&pl.r2c));
        CUFFT_CK(cufftCreate(&pl.c2r));
        it = plans.emplace(n, pl).first;   // owned from here on (reset() destroys them)
        CUFFT_CK(cufftSetAutoAllocation(pl.r2c, 0));
        CUFFT_CK(cufftSetAutoAllocation(pl.c2r, 0));
        CUFFT_CK(cufftMakePlanMany(pl.r2c, 1, nn, inembed, (int)S, 1, onembed, (int)S, 1, CUFFT_R2C, (int)S, &ws_a));
        CUFFT_CK(cufftMakePlanMany(pl.c2r, 1, nn, onembed, (int)S, 1, inembed, (int)S, 1, CUFFT_C2R, (int)S, &ws_b));
        CUFFT_CK(cufftSetStream(pl.r2c, ctx.stream));
        CUFFT_CK(cufftSetStream(pl.c2r, ctx.stream));
        it->second.work_bytes = std::max(ws_a, ws_b);
        if (it->second.work_bytes > fft_work_bytes) {
            if (fft_work) arena.free_block(fft_work);
            fft_work = nullptr;
            fft_work_bytes = 0;
            MCK(arena.alloc_bytes(&fft_work, it->second.work_bytes));
            fft_work_bytes = it->second.work_bytes;
            for (auto& kv : plans) kv.second.bound = nullptr;
        }
    }
    if (it->second.bound != fft_work) {
        if (fft_work) {
            CUFFT_CK(cufftSetWorkArea(it->second.r2c, fft_work));
            CUFFT_CK(cufftSetWorkArea(it->second.c2r, fft_work));
        }
        it->second.bound = fft_work;
    }
    const cufftHandle plan_r2c = it->second.r2c, plan_c2r = it->second.c2r;
    double mask_fl = 0, mask_fh = 0;
    {
        double lo = p.coLow, hi = p.coHigh;
        if (lo == 0.0) lo += 0.01;  // TemporalFilter.cpp:26-27
        // createIdealBandpassFilter (TemporalFilter.cpp:59-80): real 0/1 mask over packed indices x,
        // read back by mulSpectrums as the complex number m[2k-1] + i m[2k] per bin (SURVEY A.4).
        const float width = (float)n;
        mask_fl = 2 * lo * width / p.framerate;
        mask_fh = 2 * hi * width / p.framerate;
    }
    {
        const bool pp = ctx.prof && ctx.prof->begin("cufft_r2c", 0, ctx.stream);
        CUFFT_CK(cufftExecR2C(plan_r2c, ring, spec));
        if (pp) ctx.prof->end(ctx.stream);
        ++*ctx.launches;
    }
    {
        const bool pp = ctx.prof && ctx.prof->begin("mask_mul", 0, ctx.stream);
        k_mask_mul<<<gs_blocks(S * (size_t)(n / 2 + 1)), 256, 0, ctx.stream>>>((float2*)spec, S, n / 2 + 1, n, mask_fl, mask_fh,
                                                                                1.0f / ((float)n * (float)n));
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    {
        const bool pp = ctx.prof && ctx.prof->begin("cufft_c2r", 0, ctx.stream);
        CUFFT_CK(cufftExecC2R(plan_c2r, spec, work));
        if (pp) ctx.prof->end(ctx.stream);
        ++*ctx.launches;
    }
    unsigned* mm = (unsigned*)minmax;
    k_mm_init<<<cdiv(4 * lanes, 256), 256, 0, ctx.stream>>>(mm, 4 * lanes);
    MCK(cudaGetLastError());
    ++*ctx.launches;
    {
        // global min/max per stream over all pixels, frames and channels (TemporalFilter.cpp:55)
        const size_t chunk = (size_t)C * small_rows;
        const int vec_ok = chunk % 4 == 0 && S % 4 == 0 && (reinterpret_cast<uintptr_t>(work) & 15) == 0;
        dim3 grid((unsigned)std::max<size_t>(1, std::min<size_t>(chunk / 1024 + 1, (size_t)(592 / lanes + 1))), lanes);
        const bool pp = ctx.prof && ctx.prof->begin("minmax_window", 0, ctx.stream);
        k_minmax<<<grid, 256, 0, ctx.stream>>>(work, chunk, n, S, mm, vec_ok);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    // the reconstructed column is logical index min(1, n-1) (MagnifyCore.hpp:189-192)
    const int logical = std::min(1, n - 1);
    const int phys = (head + logical) % ring_mod;
    {
        const bool pp = ctx.prof && ctx.prof->begin("select", 0, ctx.stream);
        k_select<<<gs_blocks(S), 256, 0, ctx.stream>>>(work + (size_t)phys * S, mm, C, ls.w, ls.h, (float)p.amplification, U[0], ulv[0].pitch, ulv[0].plane, planes);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    // pyrUp chain with default 2x sizes, then bilinear resize to the frame size (SpatialFilter.cpp:40-50)
    for (int i = 0; i < levels; ++i) {
        const Level& s0 = ulv[(size_t)i];
        const Level& d0 = ulv[(size_t)i + 1];
        dim3 grid(cdiv(d0.w, 64), cdiv(d0.h, 32), planes);
        const bool pp = ctx.prof && ctx.prof->begin("pyrup2x", i, ctx.stream);
        k_pyrup2x<<<grid, 256, 0, ctx.stream>>>(s0, d0, U[(size_t)i], U[(size_t)i + 1]);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    const float* color_img = U[(size_t)levels];
    if (U[(size_t)levels + 1]) {
        dim3 grid(cdiv(w, 256), h, planes);
        const bool pp = ctx.prof && ctx.prof->begin("resize", 0, ctx.stream);
        k_resize_linear<<<grid, 256, 0, ctx.stream>>>(ulv[(size_t)levels], lv[0], U[(size_t)levels], U[(size_t)levels + 1]);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
        color_img = U[(size_t)levels + 1];
    }
    {
        dim3 grid((unsigned)std::max(1, std::min(C * h, 1184 / lanes + 1)), lanes);
        const bool pp = ctx.prof && ctx.prof->begin("minmax_out", 0, ctx.stream);
        k_sum_minmax<<<grid, 256, 0, ctx.stream>>>(G[0], color_img, lv[0], C, mm + 2 * lanes);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    {
        dim3 grid(cdiv(w, 256), h, lanes);
        const bool pp = ctx.prof && ctx.prof->begin("color_egress", 0, ctx.stream);
        if (C == 3) k_color_egress<3><<<grid, 256, 0, ctx.stream>>>(G[0], color_img, lv[0], mm + 2 * lanes, io.out, io.out_step, io.out_lane_stride, ctx.float_out);
        else k_color_egress<1><<<grid, 256, 0, ctx.stream>>>(G[0], color_img, lv[0], mm + 2 * lanes, io.out, io.out_step, io.out_lane_stride, ctx.float_out);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    *produced = 1;
    return MC_OK;
}

void ColorMode::find_state(const char*, int, StateRef& out) { out = StateRef{}; }

}  // namespace mc
