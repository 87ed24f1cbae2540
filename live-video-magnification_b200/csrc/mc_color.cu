// Color mode — device twin of magcore::magnifyColor (reference
// src/processing/magnification/MagnifyCore.hpp:163-206): Gaussian pyrDown chain, rolling temporal
// window kept as a device ring buffer, ideal band-pass along time with cuFFT (R2C -> CCS-mask
// multiply -> C2R), global min-max normalisation, pyrUp chain (+ bilinear resize), min-max stretch.
#include <cfloat>
#include <cmath>
#include <algorithm>
#include <cassert>
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

// small pyramid level (pitched planes) -> one time slot of the ring, rows packed tight, each lane's block followed by
// `pad` floats.  With a lane table each lane goes to its own slot, and held lanes are skipped.
__global__ void k_ring_append(const float* __restrict__ src, int w, int h, int pitch, size_t plane,
                              float* __restrict__ ring, size_t S, int pad, int slot, int planes, int C,
                              const ColorLane* __restrict__ tab) {
    const size_t n = (size_t)planes * h * w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int pl = (int)(i / ((size_t)h * w));
        const int rem = (int)(i - (size_t)pl * h * w);
        const int y = rem / w, x = rem - y * w;
        size_t o = (size_t)slot * S + i;
        if (tab || pad) {   // uniform over the launch: the lock-step path has no per-element lane lookup
            const int lane = pl / C;
            const int s = tab ? tab[lane].append : slot;
            if (s < 0) continue;
            o = (size_t)s * S + i + (size_t)lane * pad;
        }
        ring[o] = src[(size_t)pl * plane + (size_t)y * pitch + x];
    }
}

// Every lane's window in logical order where its ring size changes, in place elsewhere: destination slot t < copy_n of
// lane blockIdx.y <- source slot (src_head + t) % src_mod.  One lane's block of a slot is `lane_sig` floats, `lstride`
// apart.
__global__ void k_ring_relayout(const float* __restrict__ src, float* __restrict__ dst, size_t S, size_t lane_sig,
                                size_t lstride, const ColorLane* __restrict__ tab) {
    const ColorLane L = tab[blockIdx.y];
    const size_t o = (size_t)blockIdx.y * lstride;
    for (int t = 0; t < L.copy_n; ++t) {
        const float* __restrict__ s = src + (size_t)((L.src_head + t) % L.src_mod) * S + o;
        float* __restrict__ d = dst + (size_t)t * S + o;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < lane_sig; i += (size_t)gridDim.x * blockDim.x) d[i] = s[i];
    }
}

// spectrum[k][i] *= mask[k]  (mulSpectrums with the CCS-packed 0/1 mask, TemporalFilter.cpp:45-48, SURVEY A.4).
// createIdealBandpassFilter (TemporalFilter.cpp:59-80) is a real 0/1 mask over the PACKED indices x (1 where
// fl <= x <= fh); mulSpectrums reads it back as the complex number m[2k-1] + i m[2k] per bin, real only for DC and
// Nyquist.  The mask is evaluated here from (fl, fh) — no host vector, no per-frame upload; `sc` carries DFT_SCALE of
// both transforms.  With a lane table each lane takes its own n, mask and scale over its first n/2+1 bins (nbins is the
// largest), and lanes that do not run the filter are skipped.
__global__ void k_mask_mul(float2* __restrict__ spec, size_t S, int nbins, int n, double fl, double fh, float sc,
                           const ColorLane* __restrict__ tab, size_t lstride) {
    const size_t total = S * nbins;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i / S);
        if (tab) {
            const ColorLane& L = tab[(i - (size_t)k * S) / lstride];
            if (L.n == 0 || 2 * k > L.n) continue;
            n = L.n; fl = L.fl; fh = L.fh; sc = L.sc;
        }
        const int xr = k == 0 ? 0 : (2 * k == n ? n - 1 : 2 * k - 1);
        const bool has_im = k != 0 && 2 * k != n;
        const float2 m = make_float2(((double)xr >= fl && (double)xr <= fh) ? sc : 0.0f,
                                     (has_im && (double)(2 * k) >= fl && (double)(2 * k) <= fh) ? sc : 0.0f);
        const float2 v = spec[i];
        spec[i] = make_float2(v.x * m.x - v.y * m.y, v.x * m.y + v.y * m.x);
    }
}

// per-lane min/max over `nchunks` chunks of `chunk` contiguous floats (chunk t at base + t*chunk_stride + lane*(chunk+pad))
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
// (TemporalFilter.cpp:55); 128-bit loads when the runs are 16-byte aligned.  blockIdx.y is the (virtual) lane v: frame
// v / lanes, whose window starts win_stride floats after the previous frame's, lane v % lanes of it.
__global__ void __launch_bounds__(256) k_minmax(const float* __restrict__ base, size_t chunk, int nchunks, size_t chunk_stride,
                                                unsigned* __restrict__ mm, int vec_ok, int pad, const ColorLane* __restrict__ tab,
                                                int lanes, size_t win_stride) {
    const int v = blockIdx.y;
    const int f = v / lanes, lane = v - f * lanes;
    if (tab) {
        nchunks = tab[v].n;
        if (nchunks == 0) return;
    }
    float mn = INFINITY, mx = -INFINITY;
    for (int t = 0; t < nchunks; ++t) {
        const float* __restrict__ p = base + (size_t)f * win_stride + (size_t)t * chunk_stride + (size_t)lane * (chunk + pad);
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
    block_minmax_commit(mn, mx, mm + 2 * v);
}

// the reconstructed column: physical slot `phys` of the filtered window, or each lane's own with a lane table.  Virtual
// lane v reads the window of frame v / lanes, win_stride = S + tstep floats after the previous frame's (tstep 0: one frame).
__global__ void k_select(const float* __restrict__ work, size_t S, int pad, int phys, const unsigned* __restrict__ mm, int C, int w, int h,
                         float alpha, float* __restrict__ dst, int pitch, size_t plane, int planes, const ColorLane* __restrict__ tab,
                         int lanes, size_t tstep) {
    const size_t n = (size_t)planes * h * w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int pl = (int)(i / ((size_t)h * w));
        const int rem = (int)(i - (size_t)pl * h * w);
        const int y = rem / w, x = rem - y * w;
        const int lane = pl / C;
        size_t o = (size_t)phys * S + i;
        if (tab || pad) {
            const int slot = tab ? tab[lane].sel : phys;
            if (slot < 0) continue;
            // i + lane * pad is lane * (lane block + pad) into the frame's slot; frame f's window adds f * tstep
            o = (size_t)slot * S + i + (size_t)lane * pad + (size_t)(lane / lanes) * tstep;
        }
        const float amp = tab ? tab[lane].amp : alpha;
        const double smin = (double)ord2f(mm[2 * lane]), smax = (double)ord2f(mm[2 * lane + 1]);
        const double scale = (smax - smin > DBL_EPSILON) ? 1.0 / (smax - smin) : 0.0;   // cv::normalize NORM_MINMAX
        const double shift = 0.0 - smin * scale;
        const float v = fmaf(work[o], (float)scale, (float)shift);
        dst[(size_t)pl * plane + (size_t)y * pitch + x] = v * amp;
    }
}

// cv::pyrUp with the default destination size 2w x 2h (SpatialFilter.cpp:45)
// kernels after the filter skip the lanes that do not produce (tab[lane].n == 0) when given a lane table
__device__ __forceinline__ bool idle_lane(const ColorLane* __restrict__ tab, int lane) { return tab && tab[lane].n == 0; }

__global__ void __launch_bounds__(256) k_pyrup2x(Level ls, Level ld, const float* __restrict__ src,
                                                 float* __restrict__ dst, const ColorLane* __restrict__ tab, int C) {
    // tile = 64 x 32 destination pixels, thread = 4 x 2 block: the 34 x 18 source window (pyrUp's border rule applied to
    // the indices) goes to shared memory once, the row pass and the column pass run in registers, 128-bit stores
    __shared__ __align__(16) float sD[18][36];
    const int plane = blockIdx.z;
    if (idle_lane(tab, plane / C)) return;
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
__global__ void k_resize_linear(Level ls, Level ld, const float* __restrict__ src, float* __restrict__ dst,
                                const ColorLane* __restrict__ tab, int C) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, plane = blockIdx.z;
    if (x >= ld.w || idle_lane(tab, plane / C)) return;
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
                                                    unsigned* __restrict__ mm, const ColorLane* __restrict__ tab) {
    // one stream per blockIdx.y; the CTAs of a stream share its C * h rows, each row read as 128-bit vectors
    const int lane = blockIdx.y;
    if (idle_lane(tab, lane)) return;
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


// out8u = convertTo(input + colorImg, 255/(max-min), -min*255/(max-min))  (MagnifyCore.hpp:202-203).  The float tap takes
// (virtual) lanes fout_v0 and up: a clip's last frame.
template <int C>
__global__ void k_color_egress(const float* __restrict__ a, const float* __restrict__ b, Level l,
                               const unsigned* __restrict__ mm, uint8_t* __restrict__ out, size_t step,
                               size_t lane_stride, float* __restrict__ fout, int fout_v0, const ColorLane* __restrict__ tab) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, lane = blockIdx.z;
    if (x >= l.w || idle_lane(tab, lane)) return;
    const double mn = (double)ord2f(mm[2 * lane]), mx = (double)ord2f(mm[2 * lane + 1]);
    const float sa = (float)(255.0 / (mx - mn)), sb = (float)(-mn * 255.0 / (mx - mn));
    uint8_t* q = out + (size_t)lane * lane_stride + (size_t)y * step + (size_t)x * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const size_t o = (size_t)(lane * C + c) * l.plane + (size_t)y * l.pitch + x;
        const float v = a[o] + b[o];
        q[c] = scaled_to_u8(v, sa, sb);
        if (fout && lane >= fout_v0) fout[(((size_t)(lane - fout_v0) * l.h + y) * l.w + x) * C + c] = v;
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
    ring = work = nullptr; spec = nullptr; minmax = nullptr; d_table = nullptr;
    allocated = false;
    count.clear(); head.clear(); mod.clear(); table.clear();
    ring_cap = 0;
    clip.arena.release();
    clip = Clip{};
    tap_frame = -1;
}

mc_status ColorMode::allocate(const ModeCtx& ctx, int width, int height, int nchannels, int nlevels) {
    reset();
    levels = nlevels; channels = nchannels; w = width; h = height;
    const int planes = lanes * channels;
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
    void* tv = nullptr;
    MCK(arena.alloc_bytes(&tv, sizeof(ColorLane) * (size_t)lanes));
    d_table = (ColorLane*)tv;
    count.assign((size_t)lanes, 0); head.assign((size_t)lanes, 0); mod.assign((size_t)lanes, 0);
    table.assign((size_t)lanes, ColorLane{});
    allocated = true;
    return MC_OK;
}

// Grows the ring to `need` slots (grow) or swaps it with `work` (a rotation); with `relayout`, lane k's slot t < copy_n
// of the new ring takes slot (src_head + t) % src_mod of the old one (d_rows[k], on the device).
mc_status ColorMode::reshape_ring(const ModeCtx& ctx, int need, bool grow, bool relayout, const ColorLane* d_rows) {
    const size_t S = slot_signals();
    float* dst = work;
    float* nwork = nullptr;
    void* nspec = nullptr;
    if (grow) {
        MCK(arena.alloc(&dst, (size_t)need * S));
        MCK(arena.alloc(&nwork, (size_t)need * S));
        MCK(arena.alloc_bytes(&nspec, sizeof(cufftComplex) * (size_t)(need / 2 + 1) * S));
    }
    if (relayout) {
        const bool pp = ctx.prof && ctx.prof->begin("ring_relayout", 0, ctx.stream);
        k_ring_relayout<<<dim3(gs_blocks(lane_sig()), (unsigned)lanes), 256, 0, ctx.stream>>>(ring, dst, S, lane_sig(), lane_stride(), d_rows);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    if (grow) {
        if (ring) {   // cudaFree orders itself after the relayout above (it synchronises the device)
            // the "filtered" tap of the last frame moves along (a load grows the ring between frames)
            MCK(cudaMemcpyAsync(nwork, work, (size_t)ring_cap * S * sizeof(float), cudaMemcpyDeviceToDevice, ctx.stream));
            arena.free_block(ring); arena.free_block(work); arena.free_block(spec);
        }
        ring = dst; work = nwork; spec = (cufftComplex*)nspec;
        ring_cap = need;
    } else {
        std::swap(ring, work);
    }
    return MC_OK;
}

// A load (mc_load_lane) whose window is longer than the ring: the ring grows as process() grows it, and every lane's
// window is copied to the slots it occupies (source slot t -> slot t), so each lane keeps its physical layout.
mc_status ColorMode::reserve_ring(const ModeCtx& ctx, int need) {
    need = std::max(need, 2);
    if (ring && ring_cap >= need) return MC_OK;
    bool has_data = false;
    std::vector<ColorLane> rows((size_t)lanes, ColorLane{});
    for (int k = 0; k < lanes; ++k) {
        need = std::max(need, mod[(size_t)k]);
        rows[(size_t)k].src_head = 0;
        rows[(size_t)k].src_mod = std::max(mod[(size_t)k], 1);
        rows[(size_t)k].copy_n = count[(size_t)k];   // head == 0 or count == mod: slots 0 .. count-1 hold the window
        has_data |= count[(size_t)k] > 0;
    }
    // pageable source: staged before the call returns; the kernels of every earlier frame that read d_table precede it
    if (has_data) MCK(cudaMemcpyAsync(d_table, rows.data(), sizeof(ColorLane) * (size_t)lanes, cudaMemcpyHostToDevice, ctx.stream));
    return reshape_ring(ctx, need, true, has_data, d_table);
}

void ColorMode::lane_planes(int lane, int lane_mod, std::vector<LanePlane>& out) const {
    out.clear();
    if (!allocated || lane_mod <= 0) return;
    // slot t of the lane is its block at t * S + lane * lstride: one 2D block of lane_mod rows
    out.push_back(LanePlane{ring + (size_t)lane * lane_stride(), slot_signals() * sizeof(float), lane_sig() * sizeof(float), (size_t)lane_mod});
}

// Grows the clip scratch to `vl` virtual lanes and `work_floats` floats of filtered windows.  The float tap is written in
// place by the last frame's egress, so the scratch holds none.
mc_status ColorMode::alloc_clip(const ModeCtx& ctx, int vl, size_t work_floats) {
    ModeCtx c = ctx;
    c.float_out = nullptr;
    MCK_ST(ClipScratch::grow(clip, c, vl, 0, 0, [&]() -> mc_status {
        const size_t vplanes = (size_t)vl * channels;
        clip.G.assign((size_t)levels + 1, nullptr);
        for (int l = 0; l <= levels; ++l) MCK(clip.arena.alloc(&clip.G[(size_t)l], vplanes * lv[(size_t)l].plane));
        clip.U.assign((size_t)levels + 2, nullptr);
        for (int i = 0; i <= levels; ++i) MCK(clip.arena.alloc(&clip.U[(size_t)i], vplanes * ulv[(size_t)i].plane));
        if (U[(size_t)levels + 1]) MCK(clip.arena.alloc(&clip.U[(size_t)levels + 1], vplanes * lv[0].plane));
        void* v = nullptr;
        MCK(clip.arena.alloc_bytes(&v, sizeof(unsigned) * 4 * (size_t)vl));
        clip.minmax = (unsigned*)v;
        MCK(clip.arena.alloc_bytes(&v, sizeof(ColorLane) * (size_t)vl));
        clip.d_table = (ColorLane*)v;
        return MC_OK;
    }));
    if (work_floats > clip.work_floats) {   // the ring grew since the scratch was made
        if (clip.work) clip.arena.free_block(clip.work);
        clip.work = nullptr;
        clip.work_floats = 0;
        MCK(clip.arena.alloc(&clip.work, work_floats));
        clip.work_floats = work_floats;
    }
    return MC_OK;
}

#define CUFFT_CK(call)                                                            \
    do {                                                                          \
        cufftResult r__ = (call);                                                 \
        if (r__ != CUFFT_SUCCESS) {                                               \
            *ctx.err = std::string(#call) + ": cufft error " + std::to_string((int)r__); \
            return MC_ERR_CUDA;                                                   \
        }                                                                         \
    } while (0)

// The R2C / C2R pair of DFT length n over every signal of a slot (plan_signals of them), or over one lane's
// channels * pixels signals (the caller offsets the pointers to the lane's block; same stride).  Plans are cached per
// (n, one_lane) and share one work area: they run one after another on the handle's stream, so warm-up costs one plan
// build per length and batch size per stream geometry instead of two cufftPlanMany + workspace malloc/free per frame.
mc_status ColorMode::fft_plan(const ModeCtx& ctx, int n, bool one_lane, FftPlans** out) {
    const int S = (int)plan_signals, batch = one_lane ? channels * small_rows : S;
    auto it = plans.find({n, one_lane});
    if (it == plans.end()) {
        FftPlans pl;
        int nn[1] = {n};
        int inembed[1] = {n}, onembed[1] = {n / 2 + 1};
        size_t ws_a = 0, ws_b = 0;
        CUFFT_CK(cufftCreate(&pl.r2c));
        CUFFT_CK(cufftCreate(&pl.c2r));
        it = plans.emplace(std::make_pair(n, one_lane), pl).first;   // owned from here on (reset() destroys them)
        CUFFT_CK(cufftSetAutoAllocation(pl.r2c, 0));
        CUFFT_CK(cufftSetAutoAllocation(pl.c2r, 0));
        CUFFT_CK(cufftMakePlanMany(pl.r2c, 1, nn, inembed, S, 1, onembed, S, 1, CUFFT_R2C, batch, &ws_a));
        CUFFT_CK(cufftMakePlanMany(pl.c2r, 1, nn, onembed, S, 1, inembed, S, 1, CUFFT_C2R, batch, &ws_b));
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
    *out = &it->second;
    return MC_OK;
}

// Append to the rolling window; once full drop the oldest column (SpatialFilter.cpp:63-84).  Then the filter's operands:
// a lane's signal is physical slots [0, n) (warming: head 0; full: n == mod), so n alone picks its DFT.  A frame call
// runs this once, a clip once per frame.
ColorMode::Step ColorMode::step(const mc_params& p0, const mc_params* lp, const std::vector<int>& want_caps, ColorLane* rows) {
    Step s;
    for (int k = 0; k < lanes; ++k) {
        const mc_params& p = lp ? lp[k] : p0;
        const double lo = p.coLow == 0.0 ? p.coLow + 0.01 : p.coLow, hi = p.coHigh;   // TemporalFilter.cpp:26-27
        const int want_cap = want_caps[(size_t)k];
        ColorLane& L = rows[k];
        int& cnt = count[(size_t)k];
        int& hd = head[(size_t)k];
        L.append = -1; L.n = 0; L.sel = -1; L.sc = 0.f; L.fl = L.fh = 0.0; L.amp = (float)p.amplification;
        if (plan.op[(size_t)k] == LANE_HOLD) continue;
        L.append = (hd + cnt) % mod[(size_t)k];
        ++cnt;
        if (cnt > want_cap && want_cap > 0) {
            hd = (hd + 1) % mod[(size_t)k];
            --cnt;
        }
        if (cnt < 2) continue;  // MagnifyCore.hpp:180 (passthrough)
        L.n = cnt;
        L.sel = (hd + std::min(1, cnt - 1)) % mod[(size_t)k];   // the reconstructed column is logical min(1, n-1) (:189-192)
        // createIdealBandpassFilter (TemporalFilter.cpp:59-80): real 0/1 mask over packed indices x, read back by
        // mulSpectrums as the complex number m[2k-1] + i m[2k] per bin (SURVEY A.4).
        const float width = (float)cnt;
        L.fl = 2 * lo * width / p.framerate;
        L.fh = 2 * hi * width / p.framerate;
        L.sc = 1.0f / ((float)cnt * (float)cnt);
        if (s.n_filter && cnt != s.n_filter) s.one_length = false;
        s.n_filter = s.n_filter ? s.n_filter : cnt;
        s.n_max = std::max(s.n_max, cnt);
    }
    // Uniform lanes (every lane appends to the same slot and filters the same columns: always so for a handle whose
    // lanes run in lock-step) take the kernels' scalar path; otherwise the kernels read the table.  Lanes with parameters
    // of their own (mask range, amplification) always read the table.
    s.uniform = plan.n_hold == 0 && !lp;
    for (int k = 1; k < lanes && s.uniform; ++k)
        s.uniform = rows[k].append == rows[0].append && rows[k].n == rows[0].n && rows[k].sel == rows[0].sel;
    return s;
}

// u8 frames of `vl` (virtual) lanes -> f32 planes g[0], and the Gaussian chain g[1 .. levels] (SpatialFilter.cpp:13-23)
mc_status ColorMode::ingest(const ModeCtx& ctx, const FrameIO& io, int vl, const std::vector<float*>& g) {
    dim3 grid(cdiv(w, 256), h, (unsigned)vl);
    const bool pp = ctx.prof && ctx.prof->begin("u8_to_planes", 0, ctx.stream);
    if (channels == 3) k_u8_to_planes<3><<<grid, 256, 0, ctx.stream>>>(io.in, io.in_step, io.in_lane_stride, w, h, g[0], lv[0].pitch, lv[0].plane);
    else k_u8_to_planes<1><<<grid, 256, 0, ctx.stream>>>(io.in, io.in_step, io.in_lane_stride, w, h, g[0], lv[0].pitch, lv[0].plane);
    if (pp) ctx.prof->end(ctx.stream);
    MCK(cudaGetLastError());
    ++*ctx.launches;
    for (int l = 0; l < levels; ++l) {
        LevelArgs a;
        a.in_kind = 0; a.g = g[(size_t)l]; a.in_plane = lv[(size_t)l].plane; a.in_row = lv[(size_t)l].pitch;
        a.channels = channels; a.lf = lv[(size_t)l]; a.lc = lv[(size_t)l + 1]; a.g_next = g[(size_t)l + 1];
        a.planes = vl * channels; a.band = 0;
        LAUNCH("gauss_down", l, launch_down(a, ctx.stream));
    }
    return MC_OK;
}

// The temporal part of one frame on the handle's ring: the append of its top Gaussian level `top` (rows: the frame's lane
// table, d_rows its device copy), then the ideal band-pass (TemporalFilter.cpp:24-57) on the physical column order into
// the window `win`, with the DFT length of each lane's window: one transform over all lanes when every filtering lane
// has the same length, else one per lane.
mc_status ColorMode::filter(const ModeCtx& ctx, const Step& s, const ColorLane* rows, const ColorLane* d_rows, const float* top,
                            float* win) {
    const Level& ls = lv[(size_t)levels];
    const int C = channels, planes = lanes * C;
    const size_t lane_sig = (size_t)C * small_rows;
    const int pad = lanes > 1 ? (int)(lane_sig & 1) : 0;
    const size_t lstride = lane_sig + pad, S = (size_t)lanes * lstride;
    const ColorLane* tab = s.uniform ? nullptr : d_rows;
    {
        const bool pp = ctx.prof && ctx.prof->begin("ring_append", 0, ctx.stream);
        k_ring_append<<<gs_blocks(S), 256, 0, ctx.stream>>>(top, ls.w, ls.h, ls.pitch, ls.plane, ring, S, pad, rows[0].append, planes, C, tab);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    if (s.n_filter == 0) return MC_OK;
    if (plan_signals != S) {
        for (auto& kv : plans) { cufftDestroy(kv.second.r2c); cufftDestroy(kv.second.c2r); }
        plans.clear();
        plan_signals = S;
    }
    auto exec = [&](bool r2c) -> mc_status {
        for (int k = 0; k < (s.one_length ? 1 : lanes); ++k) {
            const int n = s.one_length ? s.n_filter : rows[k].n;
            if (n == 0) continue;
            FftPlans* pl = nullptr;
            MCK_ST(fft_plan(ctx, n, !s.one_length, &pl));
            const size_t o = s.one_length ? 0 : (size_t)k * lstride;
            const bool pp = ctx.prof && ctx.prof->begin(r2c ? "cufft_r2c" : "cufft_c2r", 0, ctx.stream);
            if (r2c) CUFFT_CK(cufftExecR2C(pl->r2c, ring + o, spec + o));
            else CUFFT_CK(cufftExecC2R(pl->c2r, spec + o, win + o));
            if (pp) ctx.prof->end(ctx.stream);
            ++*ctx.launches;
        }
        return MC_OK;
    };
    MCK_ST(exec(true));
    {
        const ColorLane& L = rows[0];   // the scalars of uniform lanes
        const bool pp = ctx.prof && ctx.prof->begin("mask_mul", 0, ctx.stream);
        k_mask_mul<<<gs_blocks(S * (size_t)(s.n_max / 2 + 1)), 256, 0, ctx.stream>>>((float2*)spec, S, s.n_max / 2 + 1, L.n, L.fl, L.fh, L.sc,
                                                                                      tab, lstride);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    return exec(false);
}

// Everything after the filter, over `vl` (virtual) lanes: frame v / lanes of virtual lane v reads its filtered window at
// win + (v / lanes) * win_stride.  row0: the scalars of uniform lanes (tab null); mm: 4 * vl slots.
mc_status ColorMode::reconstruct(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int vl, const ColorLane& row0,
                                 const ColorLane* tab, const std::vector<float*>& g, const std::vector<float*>& u, const float* win,
                                 size_t win_stride, unsigned* mm, int fout_v0) {
    const Level& ls = lv[(size_t)levels];
    const int C = channels, vplanes = vl * C;
    const size_t lane_sig = (size_t)C * small_rows;
    const int pad = lanes > 1 ? (int)(lane_sig & 1) : 0;
    const size_t S = (size_t)lanes * (lane_sig + pad);
    k_mm_init<<<cdiv(4 * vl, 256), 256, 0, ctx.stream>>>(mm, 4 * vl);
    MCK(cudaGetLastError());
    ++*ctx.launches;
    {
        // global min/max per stream over all pixels, frames and channels (TemporalFilter.cpp:55)
        const size_t chunk = lane_sig;
        const int vec_ok = chunk % 4 == 0 && S % 4 == 0 && win_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(win) & 15) == 0;
        dim3 grid((unsigned)std::max<size_t>(1, std::min<size_t>(chunk / 1024 + 1, (size_t)(592 / vl + 1))), (unsigned)vl);
        const bool pp = ctx.prof && ctx.prof->begin("minmax_window", 0, ctx.stream);
        k_minmax<<<grid, 256, 0, ctx.stream>>>(win, chunk, row0.n, S, mm, vec_ok, pad, tab, lanes, win_stride);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    {
        const bool pp = ctx.prof && ctx.prof->begin("select", 0, ctx.stream);
        k_select<<<gs_blocks((size_t)(vl / lanes) * S), 256, 0, ctx.stream>>>(win, S, pad, row0.sel, mm, C, ls.w, ls.h, (float)p.amplification,
                                                                              u[0], ulv[0].pitch, ulv[0].plane, vplanes, tab, lanes,
                                                                              win_stride - S);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    // pyrUp chain with default 2x sizes, then bilinear resize to the frame size (SpatialFilter.cpp:40-50)
    for (int i = 0; i < levels; ++i) {
        const Level& s0 = ulv[(size_t)i];
        const Level& d0 = ulv[(size_t)i + 1];
        dim3 grid(cdiv(d0.w, 64), cdiv(d0.h, 32), (unsigned)vplanes);
        const bool pp = ctx.prof && ctx.prof->begin("pyrup2x", i, ctx.stream);
        k_pyrup2x<<<grid, 256, 0, ctx.stream>>>(s0, d0, u[(size_t)i], u[(size_t)i + 1], tab, C);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    const float* color_img = u[(size_t)levels];
    if (u[(size_t)levels + 1]) {
        dim3 grid(cdiv(w, 256), h, (unsigned)vplanes);
        const bool pp = ctx.prof && ctx.prof->begin("resize", 0, ctx.stream);
        k_resize_linear<<<grid, 256, 0, ctx.stream>>>(ulv[(size_t)levels], lv[0], u[(size_t)levels], u[(size_t)levels + 1], tab, C);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
        color_img = u[(size_t)levels + 1];
    }
    {
        dim3 grid((unsigned)std::max(1, std::min(C * h, 1184 / vl + 1)), (unsigned)vl);
        const bool pp = ctx.prof && ctx.prof->begin("minmax_out", 0, ctx.stream);
        k_sum_minmax<<<grid, 256, 0, ctx.stream>>>(g[0], color_img, lv[0], C, mm + 2 * vl, tab);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    {
        dim3 grid(cdiv(w, 256), h, (unsigned)vl);
        const bool pp = ctx.prof && ctx.prof->begin("color_egress", 0, ctx.stream);
        if (C == 3) k_color_egress<3><<<grid, 256, 0, ctx.stream>>>(g[0], color_img, lv[0], mm + 2 * vl, io.out, io.out_step, io.out_lane_stride, ctx.float_out, fout_v0, tab);
        else k_color_egress<1><<<grid, 256, 0, ctx.stream>>>(g[0], color_img, lv[0], mm + 2 * vl, io.out, io.out_step, io.out_lane_stride, ctx.float_out, fout_v0, tab);
        if (pp) ctx.prof->end(ctx.stream);
        MCK(cudaGetLastError());
        ++*ctx.launches;
    }
    return MC_OK;
}

mc_status ColorMode::process(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int nlevels, int* produced, int frames) {
    *produced = 0;
    want_cap.resize((size_t)lanes);
    for (int k = 0; k < lanes; ++k)   // MagnifyCore.hpp:176, from each lane's own frame rate
        want_cap[(size_t)k] = optimal_buffer_size((int)(ctx.lane_params ? ctx.lane_params[k] : p).framerate);
    const int planes = lanes * io.channels;
    if (!allocated) MCK_ST(allocate(ctx, io.w, io.h, io.channels, nlevels));
    plan.make(ctx.lane_ops, lanes, false);
    if (plan.n_hold == lanes) return MC_OK;   // nothing to append, nothing produced
    const size_t S = slot_signals();

    // Ring geometry, lane by lane.  A lane's `mod` is its LOGICAL ring size (its slots are taken modulo it), `ring_cap`
    // the allocation.  It follows the window cap the frame rate asks for; when that changes (rare: a UI action) the
    // lane's window is laid out once in logical order — into a bigger allocation when needed, the replaced buffers
    // being freed — so that "head == 0 or count == mod" holds from then on and no per-frame compaction is ever needed.
    // A window that is longer than a lowered cap keeps its length, as the reference's does (it drops one column per
    // appended column, SpatialFilter.cpp:73-83).  A held lane is not touched: its window and slots stay as they are.
    // Every other lane keeps its physical slots, so each lane's layout is that of a 1-lane handle fed its frames.
    int need = 2;
    bool rotate = false, has_data = false;
    for (int k = 0; k < lanes; ++k) {
        ColorLane& L = table[(size_t)k];
        if (plan.op[(size_t)k] == LANE_FIRST) count[(size_t)k] = head[(size_t)k] = 0;   // the lane's window restarts empty
        const int want_mod = std::max(std::max(want_cap[(size_t)k], count[(size_t)k]), 2);
        L.src_head = 0; L.src_mod = std::max(mod[(size_t)k], 1); L.copy_n = count[(size_t)k];
        if (plan.op[(size_t)k] != LANE_HOLD && want_mod != mod[(size_t)k]) {
            L.src_head = head[(size_t)k];
            rotate |= head[(size_t)k] != 0;
            head[(size_t)k] = 0;
            mod[(size_t)k] = want_mod;
        }
        need = std::max(need, mod[(size_t)k]);
        has_data |= count[(size_t)k] > 0;
    }
    const bool grow = ring == nullptr || ring_cap < need;
    const bool relayout = (grow || rotate) && has_data;

    // The append and filter rules, frame by frame: a frame call's rows are `table`, a clip's the rows of every virtual
    // lane.  The clip's restarts and ring geometry are those of its first frame; with constant params a lane's logical
    // ring size cannot change after that (its window grows to the cap or, above a lowered cap, keeps its length).
    const int vl = frames * lanes;
    const size_t win_stride = ((size_t)need * S + 63) / 64 * 64;   // a clip's filtered windows, 256-byte aligned
    ColorLane* rows = table.data();
    Step s1;
    if (frames > 1) {
        MCK_ST(alloc_clip(ctx, vl, (size_t)frames * win_stride));
        clip.table.assign((size_t)vl, ColorLane{});
        clip.steps.assign((size_t)frames, Step{});
        std::copy(table.begin(), table.end(), clip.table.begin());   // frame 0's relayout fields
        rows = clip.table.data();
    }
    for (int t = 0; t < frames; ++t) {
        for (int k = 0; t > 0 && k < lanes; ++k)
            assert(plan.op[(size_t)k] == LANE_HOLD || std::max(std::max(want_cap[(size_t)k], count[(size_t)k]), 2) == mod[(size_t)k]);
        (frames > 1 ? clip.steps[(size_t)t] : s1) = step(p, ctx.lane_params, want_cap, rows + (size_t)t * lanes);
    }
    ColorLane* dtab = frames > 1 ? clip.d_table : d_table;
    // pageable source: staged before the call returns; stream-ordered after the previous frame's kernels read the table
    if (frames > 1 || relayout || !s1.uniform)
        MCK(cudaMemcpyAsync(dtab, rows, sizeof(ColorLane) * (size_t)vl, cudaMemcpyHostToDevice, ctx.stream));

    if (grow || rotate) MCK_ST(reshape_ring(ctx, need, grow, relayout, dtab));

    if (frames == 1) {
        tap_frame = -1;
        MCK_ST(ingest(ctx, io, lanes, G));
        MCK_ST(filter(ctx, s1, rows, d_table, G[(size_t)levels], work));
        if (s1.n_filter == 0) return MC_OK;
        MCK_ST(reconstruct(ctx, io, p, lanes, table[0], s1.uniform ? nullptr : d_table, G, U, work, S, (unsigned*)minmax, 0));
        for (int k = 0; k < lanes; ++k) ctx.lane_produced[(size_t)k] = table[(size_t)k].n > 0 ? 1 : 0;
        *produced = 1;
        return MC_OK;
    }

    // A clip: the per-frame kernels once over every virtual lane, the temporal part frame by frame on the ring exactly as
    // frame calls run it (same plans, operands and layout), each frame's filtered window kept for the kernels after it.
    tap_frame = frames - 1;
    clip.win_stride = win_stride;
    MCK_ST(ingest(ctx, io, vl, clip.G));
    const Level& ls = lv[(size_t)levels];
    bool any = false;
    for (int t = 0; t < frames; ++t) {
        const Step& s = clip.steps[(size_t)t];
        MCK_ST(filter(ctx, s, rows + (size_t)t * lanes, dtab + (size_t)t * lanes, clip.G[(size_t)levels] + (size_t)t * planes * ls.plane,
                      clip.work + (size_t)t * win_stride));
        any |= s.n_filter > 0;
    }
    if (any) MCK_ST(reconstruct(ctx, io, p, vl, rows[0], dtab, clip.G, clip.U, clip.work, win_stride, clip.minmax, vl - lanes));
    for (int v = 0; v < vl; ++v) ctx.lane_produced[(size_t)v] = rows[v].n > 0 ? 1 : 0;
    *produced = any ? 1 : 0;
    std::copy(rows + (size_t)(vl - lanes), rows + vl, table.begin());   // the taps read the last frame's rows
    return MC_OK;
}

// Read-only taps on the buffers of the last frame call or of a clip's last frame (include/magcore_b200.h, at mc_get_state).  A column of "window" or
// "filtered" is served only while every lane has it, "filtered" and "up" only while every lane ran the filter.
void ColorMode::find_state(const char* name, int level, StateRef& out) {
    out = StateRef{};
    if (!allocated || level < 0) return;
    int have = count[0], filt = table[0].n;   // columns every lane has / every lane filtered
    for (int k = 1; k < lanes; ++k) {
        have = std::min(have, count[(size_t)k]);
        filt = std::min(filt, table[(size_t)k].n);
    }
    const std::string nm(name);
    out.channels = channels; out.read_only = true;
    // after a clip the per-frame planes are its last frame's in the clip scratch
    auto frame_planes = [&](const std::vector<float*>& own, const std::vector<float*>& clipped, int l, const Level& lvl) {
        return tap_frame < 0 ? own[(size_t)l] : clipped[(size_t)l] + (size_t)tap_frame * lanes * channels * lvl.plane;
    };
    auto planes_of = [&](float* p, const Level& l) {
        out.ptr = p; out.rows = l.h; out.cols = l.w; out.pitch = l.pitch; out.plane_stride = l.plane;
    };
    if (nm == "gauss") {
        if (level <= levels && *std::max_element(count.begin(), count.end()) > 0) planes_of(frame_planes(G, clip.G, level, lv[(size_t)level]), lv[(size_t)level]);
    } else if (nm == "up") {
        if (filt >= 2 && level <= levels) planes_of(frame_planes(U, clip.U, level, ulv[(size_t)level]), ulv[(size_t)level]);
        else if (filt >= 2 && level == levels + 1 && U[(size_t)level]) planes_of(frame_planes(U, clip.U, level, lv[0]), lv[0]);
    } else if (nm == "window" || nm == "filtered") {
        const bool win = nm == "window";
        if (level >= (win ? have : filt)) return;
        // a slot holds every lane's block of channels * pixels tightly packed signals, odd blocks of a multi-lane handle
        // followed by one padding float (process()); logical column `level` of a lane is its slot (head + level) % mod
        const Level& ls = lv[(size_t)levels];
        const size_t lane_sig = (size_t)channels * small_rows, lstride = lane_sig + (lanes > 1 ? (lane_sig & 1) : 0);
        out.ptr = win ? ring : tap_frame < 0 ? work : clip.work + (size_t)tap_frame * clip.win_stride;
        out.rows = ls.h; out.cols = ls.w; out.pitch = ls.w; out.plane_stride = (size_t)small_rows;
        for (int k = 0; k < lanes; ++k)
            out.lane_off.push_back((size_t)((head[(size_t)k] + level) % mod[(size_t)k]) * lanes * lstride + (size_t)k * lstride);
    }
}

}  // namespace mc
