// Phase (Riesz) mode — device twin of magcore::magnifyRiesz (reference
// src/processing/magnification/MagnifyCore.hpp:209-279) with RieszPyramid.cpp / TemporalFilter.cpp:299-362.
//
//   analysis : 9x9 high-pass band + 9x9 2*low-pass, subsampled            (RieszPyramid.cpp:215-238)
//   phase    : Riesz pair (1x5 / 5x1) + quaternionic phase difference +
//              amplitude + both 2nd-order Butterworth IIRs (DF-II)         (RieszPyramid.cpp:66-111, TemporalFilter.cpp:340-351)
//   amplify  : separable 13-tap Gaussian of (A, cos, sin) + phase shift    (RieszPyramid.cpp:114-144)
//   collapse : zero-injected 2*LP up-sampling + HP of the band, summed     (RieszPyramid.cpp:304-325)
//   egress   : merge L' with a,b -> Lab2BGR -> u8                           (MagnifyCore.hpp:272-276)
//
// The point-wise quaternion algebra uses explicit round-to-nearest intrinsics (no FMA contraction)
// so that, given identical inputs, it rounds exactly like OpenCV's element-wise cv::multiply / add /
// divide / sqrt calls — acos near 1 is ill-conditioned (SURVEY.md A.7).
#include <cmath>
#include <cstring>

#include "mc_modes.h"
#include "mc_tma.cuh"

namespace mc {

namespace {

// literal 4-decimal tap tables of the Riesz-pyramid paper, as the reference writes them
// (RieszPyramid.cpp:146-167); the low-pass is used x2 on analysis and synthesis (:232, :316).
__constant__ float c_hp[81] = {
    0.0000f, 0.0003f, 0.0011f, 0.0022f, 0.0027f, 0.0022f, 0.0011f, 0.0003f, 0.0000f,
    0.0003f, 0.0020f, 0.0059f, 0.0103f, 0.0123f, 0.0103f, 0.0059f, 0.0020f, 0.0003f,
    0.0011f, 0.0059f, 0.0151f, 0.0249f, 0.0292f, 0.0249f, 0.0151f, 0.0059f, 0.0011f,
    0.0022f, 0.0103f, 0.0249f, 0.0402f, 0.0469f, 0.0402f, 0.0249f, 0.0103f, 0.0022f,
    0.0027f, 0.0123f, 0.0292f, 0.0469f, -0.9455f, 0.0469f, 0.0292f, 0.0123f, 0.0027f,
    0.0022f, 0.0103f, 0.0249f, 0.0402f, 0.0469f, 0.0402f, 0.0249f, 0.0103f, 0.0022f,
    0.0011f, 0.0059f, 0.0151f, 0.0249f, 0.0292f, 0.0249f, 0.0151f, 0.0059f, 0.0011f,
    0.0003f, 0.0020f, 0.0059f, 0.0103f, 0.0123f, 0.0103f, 0.0059f, 0.0020f, 0.0003f,
    0.0000f, 0.0003f, 0.0011f, 0.0022f, 0.0027f, 0.0022f, 0.0011f, 0.0003f, 0.0000f,
};
__constant__ float c_lp[81] = {
    -0.0001f, -0.0007f, -0.0023f, -0.0046f, -0.0057f, -0.0046f, -0.0023f, -0.0007f, -0.0001f,
    -0.0007f, -0.0030f, -0.0047f, -0.0025f, -0.0003f, -0.0025f, -0.0047f, -0.0030f, -0.0007f,
    -0.0023f, -0.0047f, 0.0054f, 0.0272f, 0.0387f, 0.0272f, 0.0054f, -0.0047f, -0.0023f,
    -0.0046f, -0.0025f, 0.0272f, 0.0706f, 0.0910f, 0.0706f, 0.0272f, -0.0025f, -0.0046f,
    -0.0057f, -0.0003f, 0.0387f, 0.0910f, 0.1138f, 0.0910f, 0.0387f, -0.0003f, -0.0057f,
    -0.0046f, -0.0025f, 0.0272f, 0.0706f, 0.0910f, 0.0706f, 0.0272f, -0.0025f, -0.0046f,
    -0.0023f, -0.0047f, 0.0054f, 0.0272f, 0.0387f, 0.0272f, 0.0054f, -0.0047f, -0.0023f,
    -0.0007f, -0.0030f, -0.0047f, -0.0025f, -0.0003f, -0.0025f, -0.0047f, -0.0030f, -0.0007f,
    -0.0001f, -0.0007f, -0.0023f, -0.0046f, -0.0057f, -0.0046f, -0.0023f, -0.0007f, -0.0001f,
};

constexpr int RT_W = 32, RT_H = 16;                 // output tile

__device__ __forceinline__ float mulr(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float addr(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float subr(float a, float b) { return __fsub_rn(a, b); }

// cv::filter2D's f32 engine (FilterVec_32f + scalar remainder; OpenCV 4.x, its AVX2 dispatch,
// tools/probe_filter2d_order.py): every output accumulates its non-zero taps in raster order — with one
// FMA per tap in the vectorised columns x < (w & ~7), with multiply-then-add in the scalar tail columns.  The device
// kernels follow that rule column by column, which makes the band planes and the Riesz pair bit-identical to the
// reference for every width (acos near 1 turns a last-ulp difference here into visible differences downstream).
__device__ __forceinline__ float f2d(float c, float v, float acc, bool tail) {
    return tail ? __fadd_rn(acc, __fmul_rn(c, v)) : fmaf(c, v, acc);
}

// 9x9 kernels are register-blocked: a thread owns a 1x4 strip, loads 12 tile values per kernel row with three
// 128-bit shared-memory reads and issues 36 FMAs on them.  Rows are dealt to warps so that both rows of a
// warp have the same parity (the sub-sampled low-pass / the zero-injected up-sampling only touch one parity),
// which keeps every parity branch warp-uniform.
constexpr int R9_W = 64, R9_H = 16;                  // output tile
constexpr int R9_SW = R9_W + 8, R9_SH = R9_H + 8;    // + 4 halo

__device__ __forceinline__ int r9_row(int tid) {     // tile row of this thread: warp w -> rows {b, b+2}, b = 4(w>>1) + (w&1)
    const int w = tid >> 5, half = (tid >> 4) & 1;
    return 4 * (w >> 1) + (w & 1) + 2 * half;
}

// Stages the (R9_SH x R9_SW) window of one plane, origin (x0-4, y0-4), BORDER_REFLECT_101.  Interior tiles with a
// tensor map: ONE cp.async.bulk.tensor copy issued by one thread, completion on an mbarrier (`bar` must have been
// initialised and fenced by the caller before the block-wide barrier that precedes this call); otherwise 128-bit loads
// (interior) or scalar reflected loads (tiles touching an image border).
__device__ __forceinline__ void r9_load_tile(float (*s)[R9_SW], const float* __restrict__ src, const Level& l, int x0, int y0,
                                             const CUtensorMap* tm = nullptr, int plane = 0, uint64_t* bar = nullptr) {
    const bool interior = x0 >= 4 && x0 + R9_W + 4 <= l.w && y0 >= 4 && y0 + R9_H + 4 <= l.h;
    if (interior && tm) {
        if (threadIdx.x == 0) {
            mbar_expect_tx(bar, R9_SH * R9_SW * sizeof(float));
            tma_load_3d(&s[0][0], tm, x0 - 4, y0 - 4, plane, bar);
        }
        mbar_wait(bar, 0);
    } else if (interior) {
        for (int i = threadIdx.x; i < R9_SH * (R9_SW / 4); i += 256) {
            const int r = i / (R9_SW / 4), c4 = i - r * (R9_SW / 4);
            *reinterpret_cast<float4*>(&s[r][4 * c4]) =
                __ldg(reinterpret_cast<const float4*>(src + (size_t)(y0 - 4 + r) * l.pitch + (x0 - 4 + 4 * c4)));
        }
    } else {
        for (int i = threadIdx.x; i < R9_SH * R9_SW; i += 256) {
            const int r = i / R9_SW, c = i - r * R9_SW;
            s[r][c] = __ldg(src + (size_t)reflect101(y0 - 4 + r, l.h) * l.pitch + reflect101(x0 - 4 + c, l.w));
        }
    }
}

// hp = filter2D(oct, HP) ; next = subsample(filter2D(oct, 2*LP))   (REFLECT_101, correlation)
__global__ void __launch_bounds__(256) k_riesz_analysis(Level l, Level ln, const float* __restrict__ oct,
                                                        float* __restrict__ hp, float* __restrict__ next,
                                                        const __grid_constant__ CUtensorMap tm, int use_tma,
                                                        const uint8_t* __restrict__ ops) {
    __shared__ __align__(128) float s[R9_SH][R9_SW];
    __shared__ __align__(8) uint64_t bar;
    const int plane = blockIdx.z;   // one plane (L) per lane
    if (lane_op(ops, plane) == LANE_HOLD) return;
    const int x0 = blockIdx.x * R9_W, y0 = blockIdx.y * R9_H;
    if (use_tma) {
        if (threadIdx.x == 0) mbar_init(&bar, 1);
        __syncthreads();
    }
    r9_load_tile(s, oct + (size_t)plane * l.plane, l, x0, y0, use_tma ? &tm : nullptr, plane, &bar);
    __syncthreads();
    const int tx = threadIdx.x & 15, y = r9_row(threadIdx.x);
    const int gy = y0 + y, gx = x0 + 4 * tx;
    if (gy >= l.h || gx >= l.w) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, lp0 = 0.f, lp1 = 0.f;
    const bool even_row = next != nullptr && !(gy & 1);   // warp-uniform
    const int tail_from = (l.w & ~7) - gx;                 // strip columns p >= tail_from are filter2D's scalar-tail columns
    if (tail_from >= 4) {
#pragma unroll
        for (int ky = 0; ky < 9; ++ky) {
            const float4 a0 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx]);
            const float4 a1 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx + 4]);
            const float4 a2 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx + 8]);
            const float v[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
#pragma unroll
            for (int kx = 0; kx < 9; ++kx) {
                const float c = c_hp[ky * 9 + kx];
#pragma unroll
                for (int p = 0; p < 4; ++p) acc[p] = fmaf(c, v[p + kx], acc[p]);
            }
            if (even_row) {
#pragma unroll
                for (int kx = 0; kx < 9; ++kx) {
                    const float c = 2.0f * c_lp[ky * 9 + kx];
                    lp0 = fmaf(c, v[kx], lp0);
                    lp1 = fmaf(c, v[2 + kx], lp1);
                }
            }
        }
    } else {   // the last strip(s) of a row whose width is not a multiple of 8
#pragma unroll
        for (int ky = 0; ky < 9; ++ky) {
            const float4 a0 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx]);
            const float4 a1 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx + 4]);
            const float4 a2 = *reinterpret_cast<const float4*>(&s[y + ky][4 * tx + 8]);
            const float v[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
#pragma unroll
            for (int kx = 0; kx < 9; ++kx) {
                const float c = c_hp[ky * 9 + kx];
#pragma unroll
                for (int p = 0; p < 4; ++p) acc[p] = f2d(c, v[p + kx], acc[p], p >= tail_from);
            }
            if (even_row) {
#pragma unroll
                for (int kx = 0; kx < 9; ++kx) {
                    const float c = 2.0f * c_lp[ky * 9 + kx];
                    lp0 = f2d(c, v[kx], lp0, 0 >= tail_from);
                    lp1 = f2d(c, v[2 + kx], lp1, 2 >= tail_from);
                }
            }
        }
    }
    float* o = hp + (size_t)plane * l.plane + (size_t)gy * l.pitch + gx;
    *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);   // rows are padded to 32 floats
    if (even_row) {
        float* q = next + (size_t)plane * ln.plane + (size_t)(gy >> 1) * ln.pitch + (gx >> 1);
        *reinterpret_cast<float2*>(q) = make_float2(lp0, lp1);                        // gx/2 is even -> 8-byte aligned; padded row
    }
}

struct Butter { double b0, b1, b2, a1, a2; };

struct PhaseArgs {
    Level l;
    const float* low;                      // this frame's band (hp)
    const float *plow, *prx, *pry;         // prior pyramid (old); null -> use this frame's (cutoff change)
    float *rx, *ry;                        // this frame's Riesz pair (written)
    float *ph_c, *ph_s;                    // accumulated phase
    float *lo_r0c, *lo_r0s, *lo_r1c, *lo_r1s, *hi_r0c, *hi_r0s, *hi_r1c, *hi_r1s;
    float *amp, *t_c, *t_s;                // amplitude, (hiIIR - loIIR) * amplitude
    Butter lo, hi;
    float* cur_low;                        // == low, written only for held lanes
    const uint8_t* ops;                    // LaneOp per lane or null
};

__device__ __forceinline__ float muld(float x, double s) { return (float)((double)x * s); }  // cv::multiply(Mat, double)

__device__ __forceinline__ float iir_step(float phase, float& r0, float& r1, const Butter& k) {
    // RieszTemporalFilter::IIRTemporalFilter (TemporalFilter.cpp:340-351), Direct Form II
    const float y = addr(muld(phase, k.b0), r0);
    r0 = subr(addr(muld(phase, k.b1), r1), muld(y, k.a1));
    r1 = subr(muld(phase, k.b2), muld(y, k.a2));
    return y;
}

// ---- the phase kernels' per-pixel arithmetic, shared by k_riesz_phase (one frame) and k_riesz_phase_clip (a clip) ----
// Both kernels evaluate the same expressions with the same round-to-nearest intrinsics, so they agree bit for bit.

// RieszPyramidLevel::build (RieszPyramid.cpp:66-78): taps [-0.2, -0.48, 0, 0.48, 0.2] around window pixel (y+2, x+2)
template <int SW>
__device__ __forceinline__ void riesz_pair(const float (*s)[SW], int y, int x, bool tail, float& rx, float& ry) {
    rx = mulr(-0.2f, s[y + 2][x]);
    rx = f2d(-0.48f, s[y + 2][x + 1], rx, tail);
    rx = f2d(0.48f, s[y + 2][x + 3], rx, tail);
    rx = f2d(0.2f, s[y + 2][x + 4], rx, tail);
    ry = mulr(-0.2f, s[y][x + 2]);
    ry = f2d(-0.48f, s[y + 1][x + 2], ry, tail);
    ry = f2d(0.48f, s[y + 3][x + 2], ry, tail);
    ry = f2d(0.2f, s[y + 4][x + 2], ry, tail);
}

// computePhaseDifferenceAndAmplitude (RieszPyramid.cpp:81-111): (low, rx, ry) against the prior (plow, prx, pry)
__device__ __forceinline__ void phase_difference(float low, float rx, float ry, float plow, float prx, float pry,
                                                 float& pd_c, float& pd_s, float& amp) {
    const float q_real = addr(addr(mulr(low, plow), mulr(rx, prx)), mulr(ry, pry));
    const float neg_low = -low;
    const float qx = addr(mulr(prx, neg_low), mulr(rx, plow));
    const float qy = addr(mulr(pry, neg_low), mulr(ry, plow));
    const float xy_sq = addr(mulr(qx, qx), mulr(qy, qy));
    const float q_amp = __fsqrt_rn(addr(mulr(q_real, q_real), xy_sq));
    const float tmp = __fdiv_rn(q_real, q_amp);
    float phi;
    if (tmp < -1.0f) phi = -1.0f;           // reference quirk: clamps to +-1.0 *radians* (RieszPyramid.cpp:15-18)
    else if (tmp > 1.0f) phi = 1.0f;
    else phi = acosf(tmp);
    const float xy_sqrt = __fsqrt_rn(xy_sq);
    pd_c = mulr(__fdiv_rn(qx, xy_sqrt), phi);
    pd_s = mulr(__fdiv_rn(qy, xy_sqrt), phi);
    if (pd_c != pd_c) pd_c = 0.f;           // cv::patchNaNs
    if (pd_s != pd_s) pd_s = 0.f;
    amp = __fsqrt_rn(q_amp);
}

// normalize(): change = highpassIIR - lowpassIIR ; result = change .* amplitude (RieszPyramid.cpp:118-120)
__device__ __forceinline__ float normalize_change(float hi, float lo, float amp) { return mulr(subr(hi, lo), amp); }

__global__ void __launch_bounds__(256) k_riesz_phase(const PhaseArgs a) {
    __shared__ float s[RT_H + 4][RT_W + 4 + 1];
    const int plane = blockIdx.z;
    const int x0 = blockIdx.x * RT_W, y0 = blockIdx.y * RT_H;
    const Level l = a.l;
    const size_t pb = (size_t)plane * l.plane;
    const int op = lane_op(a.ops, plane);
    if (op != LANE_RUN) {
        for (int i = threadIdx.x; i < RT_H * RT_W; i += 256) {
            const int gy = y0 + i / RT_W, gx = x0 + i % RT_W;
            if (gy >= l.h || gx >= l.w) continue;
            const size_t o = pb + (size_t)gy * l.pitch + gx;
            if (op == LANE_HOLD) {
                // the cur <-> old swap after this kernel must hand the held lane its `old` pyramid back unchanged
                if (a.plow) { a.cur_low[o] = a.plow[o]; a.rx[o] = a.prx[o]; a.ry[o] = a.pry[o]; }
            } else {
                // the lane's first frame (RieszPyramid.cpp:196-213, MagnifyCore.hpp:226-240): `old` becomes this frame's
                // band with a zero Riesz pair, the phases and both filters' registers start at zero
                a.rx[o] = 0.f; a.ry[o] = 0.f;
                a.ph_c[o] = 0.f; a.ph_s[o] = 0.f;
                a.lo_r0c[o] = 0.f; a.lo_r0s[o] = 0.f; a.lo_r1c[o] = 0.f; a.lo_r1s[o] = 0.f;
                a.hi_r0c[o] = 0.f; a.hi_r0s[o] = 0.f; a.hi_r1c[o] = 0.f; a.hi_r1s[o] = 0.f;
            }
        }
        return;
    }
    for (int i = threadIdx.x; i < (RT_H + 4) * (RT_W + 4); i += 256) {
        const int r = i / (RT_W + 4), c = i - r * (RT_W + 4);
        s[r][c] = __ldg(a.low + pb + (size_t)reflect101(y0 - 2 + r, l.h) * l.pitch + reflect101(x0 - 2 + c, l.w));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < RT_H * RT_W; i += 256) {
        const int y = i / RT_W, x = i - y * RT_W;
        const int gy = y0 + y, gx = x0 + x;
        if (gy >= l.h || gx >= l.w) continue;
        const size_t o = pb + (size_t)gy * l.pitch + gx;
        const float low = s[y + 2][x + 2];
        const bool tail = gx >= (l.w & ~7);     // filter2D's scalar-tail columns, see f2d()
        float rx, ry;
        riesz_pair(s, y, x, tail, rx, ry);
        a.rx[o] = rx;
        a.ry[o] = ry;
        const float plow = a.plow ? a.plow[o] : low;
        const float prx = a.plow ? a.prx[o] : rx;
        const float pry = a.plow ? a.pry[o] : ry;
        float pd_c, pd_s, amp;
        phase_difference(low, rx, ry, plow, prx, pry, pd_c, pd_s, amp);
        // temporal band-pass of the accumulated phase (MagnifyCore.hpp:259-264)
        const float ph_c = addr(a.ph_c[o], pd_c), ph_s = addr(a.ph_s[o], pd_s);
        a.ph_c[o] = ph_c;
        a.ph_s[o] = ph_s;
        float r0, r1;
        r0 = a.lo_r0c[o]; r1 = a.lo_r1c[o];
        const float lo_c = iir_step(ph_c, r0, r1, a.lo);
        a.lo_r0c[o] = r0; a.lo_r1c[o] = r1;
        r0 = a.lo_r0s[o]; r1 = a.lo_r1s[o];
        const float lo_s = iir_step(ph_s, r0, r1, a.lo);
        a.lo_r0s[o] = r0; a.lo_r1s[o] = r1;
        r0 = a.hi_r0c[o]; r1 = a.hi_r1c[o];
        const float hi_c = iir_step(ph_c, r0, r1, a.hi);
        a.hi_r0c[o] = r0; a.hi_r1c[o] = r1;
        r0 = a.hi_r0s[o]; r1 = a.hi_r1s[o];
        const float hi_s = iir_step(ph_s, r0, r1, a.hi);
        a.hi_r0s[o] = r0; a.hi_r1s[o] = r1;
        a.amp[o] = amp;
        a.t_c[o] = normalize_change(hi_c, lo_c, amp);
        a.t_s[o] = normalize_change(hi_s, lo_s, amp);
    }
}

// ------------------------------------------------------------------------------------------------
// phase_clip: k_riesz_phase over a clip of `frames` consecutive frames of every lane.  The grid is k_riesz_phase's over
// the handle's `lanes` state planes.  Each thread keeps the temporal state of its two pixels in registers from the first
// frame to the last: the prior {low, Rx, Ry}, both phase accumulators and the 8 DF-II registers.  The state then moves
// once per clip instead of once per frame.  Per frame t the CTA stages the band window of virtual plane t * lanes + k and
// writes that plane's Riesz pair and (amp, t_c, t_s).  With USE_TMA an interior tile requests the window of frame t+1
// into the second buffer while frame t is computed; border tiles keep the reflected loads.
// ------------------------------------------------------------------------------------------------
// band window: the 2-pixel halo, widened to origin (x0-4, y0-2) so that a TMA box starts on a 16-byte boundary: 40 x 20
constexpr int RT_SW = RT_W + 8, RT_SH = RT_H + 4;

struct PhaseClipArgs {
    Level l;
    const float* band;                     // every frame's band (virtual plane t * lanes + k)
    float *rx, *ry;                        // every frame's Riesz pair (written; null under analysis_only)
    float *amp, *t_c, *t_s;                // every frame's amplitude and (hiIIR - loIIR) * amplitude (likewise)
    float *old_low, *old_rx, *old_ry;      // prior pyramid: read at the clip's start, the last frame's written at its end
    float *ph_c, *ph_s;                    // accumulated phase
    float *lo_r0c, *lo_r0s, *lo_r1c, *lo_r1s, *hi_r0c, *hi_r0s, *hi_r1c, *hi_r1s;
    Butter lo, hi;
    int first;                             // every lane's first frame is the clip's first frame
    int rebuild_old;                       // cutoff change: frame 0's prior is frame 0 itself
    const uint8_t* ops;                    // LaneOp per lane at the clip's first frame, or null
};

template <bool USE_TMA>
__global__ void __launch_bounds__(256) k_riesz_phase_clip(const PhaseClipArgs a, const int frames, const int lanes,
                                                          const __grid_constant__ CUtensorMap tm) {
    __shared__ __align__(128) float s0[RT_SH][RT_SW];
    __shared__ __align__(128) float s1[USE_TMA ? RT_SH : 1][RT_SW];
    __shared__ __align__(8) uint64_t bar[2];
    const int lane = blockIdx.z;
    const int op = lane_op(a.ops, lane);
    if (op == LANE_HOLD) return;                     // held lane: skipped for the whole clip
    const bool first = a.first || op == LANE_FIRST;  // the lane's first frame is the clip's first frame
    const int x0 = blockIdx.x * RT_W, y0 = blockIdx.y * RT_H;
    const Level l = a.l;
    const bool tma = USE_TMA && x0 >= 4 && x0 + RT_W + 4 <= l.w && y0 >= 2 && y0 + RT_H + 2 <= l.h;   // CTA-uniform
    const int x = threadIdx.x % RT_W, yt = threadIdx.x / RT_W;   // pixels (yt, x) and (yt + 8, x) of the tile
    const int gx = x0 + x;
    const bool tail = gx >= (l.w & ~7);   // filter2D's scalar-tail columns, see f2d()

    float plow[2], prx[2], pry[2], pc[2], ps[2], lr0c[2], lr0s[2], lr1c[2], lr1s[2], hr0c[2], hr0s[2], hr1c[2], hr1s[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int gy = y0 + yt + 8 * j;
        const bool ld = !first && gy < l.h && gx < l.w;   // a first frame starts from zero phases and registers
        const size_t o = (size_t)lane * l.plane + (size_t)gy * l.pitch + gx;
        plow[j] = ld ? a.old_low[o] : 0.f; prx[j] = ld ? a.old_rx[o] : 0.f; pry[j] = ld ? a.old_ry[o] : 0.f;
        pc[j] = ld ? a.ph_c[o] : 0.f; ps[j] = ld ? a.ph_s[o] : 0.f;
        lr0c[j] = ld ? a.lo_r0c[o] : 0.f; lr0s[j] = ld ? a.lo_r0s[o] : 0.f; lr1c[j] = ld ? a.lo_r1c[o] : 0.f; lr1s[j] = ld ? a.lo_r1s[o] : 0.f;
        hr0c[j] = ld ? a.hi_r0c[o] : 0.f; hr0s[j] = ld ? a.hi_r0s[o] : 0.f; hr1c[j] = ld ? a.hi_r1c[o] : 0.f; hr1s[j] = ld ? a.hi_r1s[o] : 0.f;
    }
    if (tma) {
        if (threadIdx.x == 0) {
            mbar_init(&bar[0], 1);
            mbar_init(&bar[1], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_expect_tx(&bar[0], RT_SH * RT_SW * sizeof(float));
            tma_load_3d(&s0[0][0], &tm, x0 - 4, y0 - 2, lane, &bar[0]);
        }
    }
    for (int t = 0; t < frames; ++t) {
        const size_t vplane = (size_t)t * lanes + lane;
        float (*s)[RT_SW] = tma && (t & 1) ? s1 : s0;
        if (tma) {
            // the other buffer was last read in frame t-1, which every thread has finished (barrier at the loop's end)
            if (threadIdx.x == 0 && t + 1 < frames) {
                uint64_t* nb = &bar[(t + 1) & 1];
                mbar_expect_tx(nb, RT_SH * RT_SW * sizeof(float));
                tma_load_3d((t & 1) ? &s0[0][0] : &s1[0][0], &tm, x0 - 4, y0 - 2, (int)(vplane + lanes), nb);
            }
            mbar_wait(&bar[t & 1], (t >> 1) & 1);
        } else {
            const float* src = a.band + vplane * l.plane;
            for (int i = threadIdx.x; i < RT_SH * RT_SW; i += 256) {
                const int r = i / RT_SW, c = i - r * RT_SW;
                s[r][c] = __ldg(src + (size_t)reflect101(y0 - 2 + r, l.h) * l.pitch + reflect101(x0 - 4 + c, l.w));
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int y = yt + 8 * j, gy = y0 + y;
            if (gy >= l.h || gx >= l.w) continue;
            const float low = s[y + 2][x + 4];   // window column x + 4 is tile column x
            if (first && t == 0) {   // the lane's first frame (see k_riesz_phase): `old` = this band with a zero pair
                plow[j] = low; prx[j] = 0.f; pry[j] = 0.f;
                continue;
            }
            float rx, ry;
            riesz_pair(s, y, x + 2, tail, rx, ry);
            const size_t o = vplane * l.plane + (size_t)gy * l.pitch + gx;
            if (a.rx) { a.rx[o] = rx; a.ry[o] = ry; }
            if (t == 0 && a.rebuild_old) { plow[j] = low; prx[j] = rx; pry[j] = ry; }
            float pd_c, pd_s, amp;
            phase_difference(low, rx, ry, plow[j], prx[j], pry[j], pd_c, pd_s, amp);
            pc[j] = addr(pc[j], pd_c);
            ps[j] = addr(ps[j], pd_s);
            const float lo_c = iir_step(pc[j], lr0c[j], lr1c[j], a.lo);
            const float lo_s = iir_step(ps[j], lr0s[j], lr1s[j], a.lo);
            const float hi_c = iir_step(pc[j], hr0c[j], hr1c[j], a.hi);
            const float hi_s = iir_step(ps[j], hr0s[j], hr1s[j], a.hi);
            if (a.amp) {
                a.amp[o] = amp;
                a.t_c[o] = normalize_change(hi_c, lo_c, amp);
                a.t_s[o] = normalize_change(hi_s, lo_s, amp);
            }
            plow[j] = low; prx[j] = rx; pry[j] = ry;   // this frame is the next one's prior
        }
        __syncthreads();   // s is refilled by the next frame
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int gy = y0 + yt + 8 * j;
        if (gy >= l.h || gx >= l.w) continue;
        const size_t o = (size_t)lane * l.plane + (size_t)gy * l.pitch + gx;
        a.old_low[o] = plow[j]; a.old_rx[o] = prx[j]; a.old_ry[o] = pry[j];
        a.ph_c[o] = pc[j]; a.ph_s[o] = ps[j];
        a.lo_r0c[o] = lr0c[j]; a.lo_r0s[o] = lr0s[j]; a.lo_r1c[o] = lr1c[j]; a.lo_r1s[o] = lr1s[j];
        a.hi_r0c[o] = hr0c[j]; a.hi_r0s[o] = hr0s[j]; a.hi_r1c[o] = hr1c[j]; a.hi_r1s[o] = hr1s[j];
    }
}

struct Gauss13 { float k[13]; };

struct AmpArgs {
    Level l;
    const float *amp, *t_c, *t_s;          // inputs to blur
    const float *low, *rx, *ry;            // this frame's band and Riesz pair
    float* out;                            // amplified band
    Gauss13 g;
    float alpha, thresh;
    const uint8_t* ops;                    // LaneOp per lane or null: only RUN lanes are amplified
};

// Tile 64 x 16, thread strip 1 x 4 (same row dealing as the 9x9 kernels is not needed here).  Row pass:
// 16 tile values -> 4 outputs per plane with three/four 128-bit shared loads; column pass likewise from the
// row-pass buffer; then the point-wise amplification on float4 global accesses.
constexpr int GA_TW = 64, GA_TH = 16;
constexpr int GA_W = GA_TW + 16, GA_H = GA_TH + 12;   // window origin (x0-8, y0-6): 8 columns of left halo keep float4 alignment

__device__ __forceinline__ float g13(const Gauss13& g, const float* v) {
    // symmetric 13-tap: centre + pairs (cv::sepFilter2D symmetric row/column filters)
    float acc = g.k[6] * v[6];
#pragma unroll
    for (int j = 1; j <= 6; ++j) acc = fmaf(g.k[6 + j], v[6 - j] + v[6 + j], acc);
    return acc;
}

__global__ void __launch_bounds__(256) k_riesz_amplify(const AmpArgs a) {
    __shared__ __align__(16) float s[3][GA_H][GA_W];
    __shared__ __align__(16) float sr[3][GA_H][GA_TW];
    const int plane = blockIdx.z;
    if (lane_op(a.ops, plane) != LANE_RUN) return;
    const int x0 = blockIdx.x * GA_TW, y0 = blockIdx.y * GA_TH;
    const Level l = a.l;
    const size_t pb = (size_t)plane * l.plane;
    const float* srcs[3] = {a.amp, a.t_c, a.t_s};
    const bool interior = x0 >= 8 && x0 + GA_TW + 8 <= l.w && y0 >= 6 && y0 + GA_TH + 6 <= l.h;
    if (interior) {
        for (int i = threadIdx.x; i < GA_H * (GA_W / 4); i += 256) {
            const int r = i / (GA_W / 4), c4 = i - r * (GA_W / 4);
            const size_t o = pb + (size_t)(y0 - 6 + r) * l.pitch + (x0 - 8 + 4 * c4);
#pragma unroll
            for (int q = 0; q < 3; ++q) *reinterpret_cast<float4*>(&s[q][r][4 * c4]) = __ldg(reinterpret_cast<const float4*>(srcs[q] + o));
        }
    } else {
        for (int i = threadIdx.x; i < GA_H * GA_W; i += 256) {
            const int r = i / GA_W, c = i - r * GA_W;
            const size_t o = pb + (size_t)reflect101(y0 - 6 + r, l.h) * l.pitch + reflect101(x0 - 8 + c, l.w);
#pragma unroll
            for (int q = 0; q < 3; ++q) s[q][r][c] = __ldg(srcs[q] + o);
        }
    }
    __syncthreads();
    // row pass: item = (row r, strip of 4 columns); output column x uses window columns x+2 .. x+14
    for (int i = threadIdx.x; i < GA_H * (GA_TW / 4); i += 256) {
        const int r = i >> 4, tx4 = (i & 15) * 4;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            float v[20];
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                const float4 t = *reinterpret_cast<const float4*>(&s[q][r][tx4 + 4 * j]);
                v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
            }
            float4 o;
            o.x = g13(a.g, v + 2); o.y = g13(a.g, v + 3); o.z = g13(a.g, v + 4); o.w = g13(a.g, v + 5);
            *reinterpret_cast<float4*>(&sr[q][r][tx4]) = o;
        }
    }
    __syncthreads();
    const int tx4 = (threadIdx.x & 15) * 4, y = threadIdx.x >> 4;
    const int gy = y0 + y, gx = x0 + tx4;
    if (gy >= l.h || gx >= l.w) return;
    float b[3][4];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        float c0[13], c1[13], c2[13], c3[13];
#pragma unroll
        for (int j = 0; j < 13; ++j) {
            const float4 t = *reinterpret_cast<const float4*>(&sr[q][y + j][tx4]);
            c0[j] = t.x; c1[j] = t.y; c2[j] = t.z; c3[j] = t.w;
        }
        b[q][0] = g13(a.g, c0); b[q][1] = g13(a.g, c1); b[q][2] = g13(a.g, c2); b[q][3] = g13(a.g, c3);
    }
    const size_t o = pb + (size_t)gy * l.pitch + gx;
    const float4 low4 = *reinterpret_cast<const float4*>(a.low + o);
    const float4 rx4 = *reinterpret_cast<const float4*>(a.rx + o);
    const float4 ry4 = *reinterpret_cast<const float4*>(a.ry + o);
    const float lowv[4] = {low4.x, low4.y, low4.z, low4.w}, rxv[4] = {rx4.x, rx4.y, rx4.z, rx4.w}, ryv[4] = {ry4.x, ry4.y, ry4.z, ry4.w};
    float outv[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        // normalize() tail + amplify() (RieszPyramid.cpp:125-143)
        const float tc = __fdiv_rn(b[1][p], b[0][p]), ts = __fdiv_rn(b[2][p], b[0][p]);
        const float mag = __fsqrt_rn(addr(mulr(tc, tc), mulr(ts, ts)));
        float m2 = mulr(mag, a.alpha);
        m2 = (m2 > a.thresh) ? a.thresh : m2;                 // THRESH_TRUNC
        float pc, ps;
        sincosf(m2, &ps, &pc);
        float pair = __fdiv_rn(addr(mulr(rxv[p], tc), mulr(ryv[p], ts)), mag);
        if (pair != pair) pair = 0.f;                          // patchNaNs
        outv[p] = subr(mulr(lowv[p], pc), mulr(pair, ps));
    }
    *reinterpret_cast<float4*>(a.out + o) = make_float4(outv[0], outv[1], outv[2], outv[3]);
}

// result_i = filter2D(injectZerosEven(nearest_up(result_{i+1})), 2*LP) + filter2D(band_i, HP)
// The zero-injected image is never materialised: only the taps that land on even/even fine positions are
// evaluated (25/20/20/16 of 81, by output parity), reading the coarse samples straight from shared memory.
constexpr int RC_CW = R9_SW / 2, RC_CH = R9_SH / 2;   // even fine positions of the window: 36 x 12

template <int PAR, bool MIXED>   // PAR = parity of the output row; MIXED: some of the strip's columns are filter2D tail columns
__device__ __forceinline__ void rc_lowpass(const float (*sc)[RC_CW], int y, int tx, int tail_from, float (&lp)[4]) {
    // output (y, x): taps ky = PAR, PAR+2, ... on coarse row (y + ky) / 2 ; kx likewise by column parity
#pragma unroll
    for (int i = 0; i < 5 - PAR; ++i) {
        const int ky = 2 * i + PAR;
        const float* row = sc[(y + ky) >> 1];
        const float2 q0 = *reinterpret_cast<const float2*>(&row[2 * tx]);
        const float2 q1 = *reinterpret_cast<const float2*>(&row[2 * tx + 2]);
        const float2 q2 = *reinterpret_cast<const float2*>(&row[2 * tx + 4]);
        const float v[6] = {q0.x, q0.y, q1.x, q1.y, q2.x, q2.y};   // coarse columns x/2 .. x/2+5 (x = 4 tx)
#pragma unroll
        for (int j = 0; j < 5; ++j) {                               // even outputs x, x+2: kx = 0,2,4,6,8
            const float c = 2.0f * c_lp[ky * 9 + 2 * j];
            lp[0] = MIXED ? f2d(c, v[j], lp[0], 0 >= tail_from) : fmaf(c, v[j], lp[0]);
            lp[2] = MIXED ? f2d(c, v[j + 1], lp[2], 2 >= tail_from) : fmaf(c, v[j + 1], lp[2]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {                               // odd outputs x+1, x+3: kx = 1,3,5,7
            const float c = 2.0f * c_lp[ky * 9 + 2 * j + 1];
            lp[1] = MIXED ? f2d(c, v[j + 1], lp[1], 1 >= tail_from) : fmaf(c, v[j + 1], lp[1]);
            lp[3] = MIXED ? f2d(c, v[j + 2], lp[3], 3 >= tail_from) : fmaf(c, v[j + 2], lp[3]);
        }
    }
}

__global__ void __launch_bounds__(256) k_riesz_collapse(Level l, Level lc, const float* __restrict__ band,
                                                        const float* __restrict__ coarse, float* __restrict__ out,
                                                        const __grid_constant__ CUtensorMap tm, int use_tma,
                                                        const uint8_t* __restrict__ ops) {
    __shared__ __align__(128) float sb[R9_SH][R9_SW];
    __shared__ __align__(16) float sc[RC_CH][RC_CW];
    __shared__ __align__(8) uint64_t bar;
    const int plane = blockIdx.z;
    if (lane_op(ops, plane) != LANE_RUN) return;
    const int x0 = blockIdx.x * R9_W, y0 = blockIdx.y * R9_H;
    if (use_tma) {
        if (threadIdx.x == 0) mbar_init(&bar, 1);
        __syncthreads();
    }
    r9_load_tile(sb, band + (size_t)plane * l.plane, l, x0, y0, use_tma ? &tm : nullptr, plane, &bar);
    const float* __restrict__ c = coarse + (size_t)plane * lc.plane;
    for (int i = threadIdx.x; i < RC_CH * RC_CW; i += 256) {
        const int r = i / RC_CW, cc = i - r * RC_CW;
        // even fine coordinates of the window (reflection keeps parity), value = coarse sample
        const int gy = reflect101(y0 - 4 + 2 * r, l.h), gx = reflect101(x0 - 4 + 2 * cc, l.w);
        sc[r][cc] = __ldg(c + (size_t)(gy >> 1) * lc.pitch + (gx >> 1));
    }
    __syncthreads();
    const int tx = threadIdx.x & 15, y = r9_row(threadIdx.x);
    const int gy = y0 + y, gx = x0 + 4 * tx;
    if (gy >= l.h || gx >= l.w) return;
    float hp[4] = {0.f, 0.f, 0.f, 0.f}, lp[4] = {0.f, 0.f, 0.f, 0.f};
    const int tail_from = (l.w & ~7) - gx;                 // see f2d(): both filter2D calls run at this level's width
    const bool mixed = tail_from < 4;
#pragma unroll
    for (int ky = 0; ky < 9; ++ky) {
        const float4 a0 = *reinterpret_cast<const float4*>(&sb[y + ky][4 * tx]);
        const float4 a1 = *reinterpret_cast<const float4*>(&sb[y + ky][4 * tx + 4]);
        const float4 a2 = *reinterpret_cast<const float4*>(&sb[y + ky][4 * tx + 8]);
        const float v[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
        if (!mixed) {
#pragma unroll
            for (int kx = 0; kx < 9; ++kx) {
                const float cf = c_hp[ky * 9 + kx];
#pragma unroll
                for (int p = 0; p < 4; ++p) hp[p] = fmaf(cf, v[p + kx], hp[p]);
            }
        } else {
#pragma unroll
            for (int kx = 0; kx < 9; ++kx) {
                const float cf = c_hp[ky * 9 + kx];
#pragma unroll
                for (int p = 0; p < 4; ++p) hp[p] = f2d(cf, v[p + kx], hp[p], p >= tail_from);
            }
        }
    }
    if (!mixed) {
        if (y & 1) rc_lowpass<1, false>(sc, y, tx, tail_from, lp);   // warp-uniform (r9_row)
        else rc_lowpass<0, false>(sc, y, tx, tail_from, lp);
    } else {
        if (y & 1) rc_lowpass<1, true>(sc, y, tx, tail_from, lp);
        else rc_lowpass<0, true>(sc, y, tx, tail_from, lp);
    }
    float* o = out + (size_t)plane * l.plane + (size_t)gy * l.pitch + gx;
    *reinterpret_cast<float4*>(o) = make_float4(addr(lp[0], hp[0]), addr(lp[1], hp[1]), addr(lp[2], hp[2]), addr(lp[3], hp[3]));
}

// merge(L', a, b) -> Lab2BGR -> u8 (MagnifyCore.hpp:272-276)
__global__ void __launch_bounds__(256) k_riesz_egress(const float* __restrict__ Lp, Level l, const int16_t* __restrict__ lab,
                                                      int pitch16, size_t plane16, const float4* __restrict__ gtab,
                                                      LabInvCoeffs coeffs, uint8_t* __restrict__ out, size_t step,
                                                      size_t lane_stride, float* __restrict__ fout, const uint8_t* __restrict__ ops) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, lane = blockIdx.z;
    if (x >= l.w || lane_op(ops, lane) != LANE_RUN) return;   // first frames pass through, held lanes are not written
    const float L = Lp[(size_t)lane * l.plane + (size_t)y * l.pitch + x];
    const int16_t* p = lab + (size_t)(lane * 3) * plane16 + (size_t)y * pitch16 + x;
    const float A = fmaf((float)p[plane16], 1.0f / 64.0f, -128.0f);
    const float B = fmaf((float)p[2 * plane16], 1.0f / 64.0f, -128.0f);
    float ob, og, orr;
    lab_to_bgr_fast<true>(L, A, B, coeffs, gtab, ob, og, orr);   // NaN L (flat regions) -> white, as OpenCV
    uint8_t* q = out + (size_t)lane * lane_stride + (size_t)y * step + (size_t)x * 3;
    q[0] = unit_to_u8(ob); q[1] = unit_to_u8(og); q[2] = unit_to_u8(orr);
    if (fout) {
        float* f = fout + (((size_t)lane * l.h + y) * l.w + x) * 3;
        f[0] = ob; f[1] = og; f[2] = orr;
    }
}

inline unsigned cdiv(int a, int b) { return (unsigned)((a + b - 1) / b); }

}  // namespace

void RieszMode::reset() {
    arena.release();
    lv.clear();
    for (auto* v : {&oct, &cur_low, &cur_rx, &cur_ry, &old_low, &old_rx, &old_ry, &phase_c, &phase_s, &lo_r0c, &lo_r0s,
                    &lo_r1c, &lo_r1s, &hi_r0c, &hi_r0s, &hi_r1c, &hi_r1s, &amp, &t_c, &t_s, &low_amp, &res})
        v->clear();
    lab16 = nullptr;
    lab16_frame = false;
    clip.arena.release();
    clip = Clip{};
    allocated = false;
}

// TemporalFilter.cpp:324-327: 2nd-order Butterworth at f / Nyquist
static void design_filter(double f, double framerate, double* A, double* B) {
    const double wn = framerate == 0.0 ? 0.0 : f / (framerate / 2.0);
    std::vector<double> a, b;
    butterworth(2, wn, a, b);
    for (int k = 0; k < 3; ++k) { A[k] = a[(size_t)k]; B[k] = b[(size_t)k]; }
}

#define KLAUNCH(name, level, ...)                                                  \
    do {                                                                           \
        const bool p__ = ctx.prof && ctx.prof->begin(name, level, ctx.stream);     \
        __VA_ARGS__;                                                               \
        if (p__) ctx.prof->end(ctx.stream);                                        \
        MCK(cudaGetLastError());                                                   \
        ++*ctx.launches;                                                           \
    } while (0)

// BGR -> Lab of io's frames (only L is magnified, MagnifyCore.hpp:217-222), then RieszPyramid::buildPyramid
// (RieszPyramid.cpp:215-238) into the octaves `octs` and the bands `bands`; the Riesz pair itself is formed in the phase
// kernel.
mc_status RieszMode::build_pyramid(const ModeCtx& ctx, const FrameIO& io, int16_t* lab, const std::vector<float*>& octs,
                                   const std::vector<float*>& bands, const std::vector<TensorMapStorage>& tm, const std::vector<char>& valid) {
    LAUNCH("lab16", 0, launch_lab16(io, *ctx.tables, lab, pitch16, plane16, ctx.stream, octs[0], lv[0].pitch, lv[0].plane));
    for (int i = 0; i < levels - 1; ++i) {
        const Level& l = lv[(size_t)i];
        dim3 grid(cdiv(l.w, R9_W), cdiv(l.h, R9_H), io.lanes);
        const int tma = ctx.opt.use_tma && valid[(size_t)i];
        KLAUNCH("riesz_analysis", i, k_riesz_analysis<<<grid, 256, 0, ctx.stream>>>(l, lv[(size_t)i + 1], octs[(size_t)i], bands[(size_t)i], octs[(size_t)i + 1],
                                                                                    *reinterpret_cast<const CUtensorMap*>(&tm[(size_t)i]), tma, io.ops));
    }
    return MC_OK;
}

// amplify (RieszPyramid.cpp:248-252) of band level i over n lanes: the blurred amplitude a and (hiIIR - loIIR) *
// amplitude tc / ts shift the phase of the band low and its Riesz pair rx / ry into `out`
mc_status RieszMode::amplify(const ModeCtx& ctx, const mc_params& p, int i, int n, const uint8_t* ops, const float* a, const float* tc,
                             const float* ts, const float* low, const float* rx, const float* ry, float* out) {
    AmpArgs m;
    m.l = lv[(size_t)i];
    m.amp = a; m.t_c = tc; m.t_s = ts;
    m.low = low; m.rx = rx; m.ry = ry;
    m.out = out;
    gaussian_kernel_13_3(m.g.k);
    m.alpha = (float)p.amplification;
    m.thresh = (float)(p.coWavelength * (3.14159265358979323846 / 100.0));  // PI_PERCENT, :214,:269
    m.ops = ops;
    dim3 grid(cdiv(m.l.w, GA_TW), cdiv(m.l.h, GA_TH), n);
    KLAUNCH("riesz_amplify", i, k_riesz_amplify<<<grid, 256, 0, ctx.stream>>>(m));
    return MC_OK;
}

// collapse (RieszPyramid.cpp:304-325) of io's frames from the residual up: level i reads its amplified band bands[i]
// and writes out[i]; then egress merges the result with a, b of `lab` into io.out (MagnifyCore.hpp:272-276)
mc_status RieszMode::collapse_egress(const ModeCtx& ctx, const FrameIO& io, const int16_t* lab, const float* residual,
                                     const std::vector<float*>& bands, const std::vector<float*>& out, const std::vector<TensorMapStorage>& tm,
                                     const std::vector<char>& valid, float* fout) {
    const float* result = residual;
    for (int i = levels - 2; i >= 0; --i) {
        const Level& l = lv[(size_t)i];
        dim3 grid(cdiv(l.w, R9_W), cdiv(l.h, R9_H), io.lanes);
        const int tma = ctx.opt.use_tma && valid[(size_t)i];
        KLAUNCH("riesz_collapse", i, k_riesz_collapse<<<grid, 256, 0, ctx.stream>>>(l, lv[(size_t)i + 1], bands[(size_t)i], result, out[(size_t)i],
                                                                                    *reinterpret_cast<const CUtensorMap*>(&tm[(size_t)i]), tma, io.ops));
        result = out[(size_t)i];
    }
    dim3 grid(cdiv(w, 256), h, io.lanes);
    KLAUNCH("riesz_egress", 0, k_riesz_egress<<<grid, 256, 0, ctx.stream>>>(result, lv[0], lab, pitch16, plane16, ctx.tables->inv_gamma, ctx.tables->inv_coeffs,
                                                                           io.out, io.out_step, io.out_lane_stride, fout, io.ops));
    return MC_OK;
}

// Cutoff changes re-design the filter, zero both filters' registers and rebuild `old` from this frame (:243-254).
mc_status RieszMode::apply_cutoffs(const ModeCtx& ctx, const mc_params& p, bool* rebuild_old) {
    auto zero_state = [&]() -> mc_status {
        *ctx.held_lost = true;   // every lane's registers are zeroed and `old` is rebuilt: a held lane restarts on release
        for (auto* v : {&phase_c, &phase_s, &lo_r0c, &lo_r0s, &lo_r1c, &lo_r1s, &hi_r0c, &hi_r0s, &hi_r1c, &hi_r1s})
            for (int i = 0; i < levels - 1; ++i)
                MCK(cudaMemsetAsync((*v)[(size_t)i], 0, (size_t)lanes * lv[(size_t)i].plane * sizeof(float), ctx.stream));
        return MC_OK;
    };
    if (lo_freq != p.coLow) {
        lo_freq = p.coLow;
        design_filter(lo_freq, framerate, loA, loB);
        MCK_ST(zero_state());
        *rebuild_old = true;
    }
    if (hi_freq != p.coHigh) {
        hi_freq = p.coHigh;
        design_filter(hi_freq, framerate, hiA, hiB);
        MCK_ST(zero_state());
        *rebuild_old = true;
    }
    return MC_OK;
}

// The handle's state for `nlevels` levels at io's size, the filters designed from p; the Riesz pair of `old`, the phases
// and the IIR registers start at zero.
mc_status RieszMode::allocate(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int nlevels) {
    reset();
    levels = nlevels; w = io.w; h = io.h;
    lv.resize((size_t)levels);
    int cw = w, ch = h;
    for (int i = 0; i < levels; ++i) {
        lv[(size_t)i] = make_level(cw, ch);
        cw = cw / 2 + (cw % 2); ch = ch / 2 + (ch % 2);   // subsample(), RieszPyramid.cpp:262-263
    }
    auto alloc_set = [&](std::vector<float*>& v, int n_levels, bool zero) -> mc_status {
        v.assign((size_t)levels, nullptr);
        for (int i = 0; i < n_levels; ++i) {
            const size_t n = (size_t)lanes * lv[(size_t)i].plane;
            MCK(arena.alloc(&v[(size_t)i], n));
            if (zero) MCK(cudaMemsetAsync(v[(size_t)i], 0, n * sizeof(float), ctx.stream));
        }
        return MC_OK;
    };
    const int nb = levels - 1;  // band levels
    MCK_ST(alloc_set(oct, levels, false));
    MCK_ST(alloc_set(cur_low, nb, false));
    for (auto* v : {&cur_rx, &cur_ry, &old_low, &amp, &t_c, &t_s, &low_amp}) MCK_ST(alloc_set(*v, nb, false));
    MCK_ST(alloc_set(res, levels, false));
    // init(): Riesz pair of `old`, phases and IIR registers start at zero (RieszPyramid.cpp:196-213, TemporalFilter.cpp:299-317)
    for (auto* v : {&old_rx, &old_ry, &phase_c, &phase_s, &lo_r0c, &lo_r0s, &lo_r1c, &lo_r1s, &hi_r0c, &hi_r0s, &hi_r1c, &hi_r1s})
        MCK_ST(alloc_set(*v, nb, true));
    // TMA descriptors for the tiles of the 9x9 kernels (option use_tma; tiles touching a border keep the reflected loads)
    tm_oct.assign((size_t)levels, TensorMapStorage{});
    tm_band.assign((size_t)levels, TensorMapStorage{});
    tm_valid.assign((size_t)levels, 0);
    for (int i = 0; i < nb; ++i)
        tm_valid[(size_t)i] = make_tensor_map_box(&tm_oct[(size_t)i], oct[(size_t)i], lv[(size_t)i], lanes, R9_SW, R9_SH) &&
                              make_tensor_map_box(&tm_band[(size_t)i], low_amp[(size_t)i], lv[(size_t)i], lanes, R9_SW, R9_SH) ? 1 : 0;
    pitch16 = round_up(w, 64);
    plane16 = (size_t)h * pitch16;
    void* lp = nullptr;
    MCK(arena.alloc_bytes(&lp, (size_t)lanes * 3 * plane16 * sizeof(int16_t)));
    lab16 = (int16_t*)lp;
    lo_freq = p.coLow; hi_freq = p.coHigh; framerate = p.framerate;
    design_filter(lo_freq, framerate, loA, loB);
    design_filter(hi_freq, framerate, hiA, hiB);
    allocated = true;
    return MC_OK;
}

mc_status RieszMode::process(const ModeCtx& ctx, const FrameIO& io_in, const mc_params& p, int nlevels, int* produced, int frames) {
    *produced = 0;
    if (io_in.channels < 3) {   // MagnifyCore.hpp:212: gray input is a silent passthrough
        lab16_frame = false;
        return MC_OK;
    }
    // Per-lane ops: lanes without state take their first frame while the others run, held lanes are skipped.  When every
    // lane is on its first frame the handle's state is rebuilt from scratch, as for the reference's first frame.
    const bool fresh = !allocated || std::isnan(loA[0]) || std::isnan(hiA[0]);  // :226
    plan.make(ctx.lane_ops, lanes, fresh);
    if (plan.n_hold == lanes) return MC_OK;   // every lane held: nothing to do
    const bool first = fresh || plan.n_first == lanes;
    if (frames > 1) {
        // A filter design that is not finite makes every frame a first frame (:226).  Such a clip runs as frame calls;
        // the design the clip's first frame leaves behind is known here: the parameters' own, at the framerate it uses.
        double A[3], B[3], C[3], D[3];
        const double fr = first ? p.framerate : framerate;
        design_filter(p.coLow, fr, A, B);
        design_filter(p.coHigh, fr, C, D);
        if (std::isnan(A[0]) || std::isnan(C[0])) return frame_loop(ctx, io_in, p, nlevels, produced, frames);
    }
    if (first) {
        if (allocated) *ctx.held_lost = true;
        MCK_ST(allocate(ctx, io_in, p, nlevels));
    }
    lab16_frame = false;   // a clip converts into its own scratch; a frame call rewrites lab16 below
    if (frames > 1) return run_clip(ctx, io_in, p, frames, first, produced);
    FrameIO io = io_in;
    MCK(plan.upload(ctx, &io.ops));
    MCK_ST(build_pyramid(ctx, io, lab16, oct, cur_low, tm_oct, tm_valid));
    lab16_frame = true;
    if (first) {
        // old = pyramid of the first frame with a zero Riesz pair; the frame itself is shown unmagnified (:239)
        for (int i = 0; i < levels - 1; ++i) std::swap(cur_low[(size_t)i], old_low[(size_t)i]);
        return MC_OK;
    }
    bool rebuild_old = false;
    MCK_ST(apply_cutoffs(ctx, p, &rebuild_old));
    const int nb = levels - 1;
    for (int i = 0; i < nb; ++i) {
        PhaseArgs a;
        a.l = lv[(size_t)i];
        a.low = cur_low[(size_t)i];
        a.plow = rebuild_old ? nullptr : old_low[(size_t)i];
        a.prx = old_rx[(size_t)i]; a.pry = old_ry[(size_t)i];
        a.rx = cur_rx[(size_t)i]; a.ry = cur_ry[(size_t)i];
        a.ph_c = phase_c[(size_t)i]; a.ph_s = phase_s[(size_t)i];
        a.lo_r0c = lo_r0c[(size_t)i]; a.lo_r0s = lo_r0s[(size_t)i]; a.lo_r1c = lo_r1c[(size_t)i]; a.lo_r1s = lo_r1s[(size_t)i];
        a.hi_r0c = hi_r0c[(size_t)i]; a.hi_r0s = hi_r0s[(size_t)i]; a.hi_r1c = hi_r1c[(size_t)i]; a.hi_r1s = hi_r1s[(size_t)i];
        a.amp = amp[(size_t)i]; a.t_c = t_c[(size_t)i]; a.t_s = t_s[(size_t)i];
        a.lo = Butter{loB[0], loB[1], loB[2], loA[1], loA[2]};
        a.hi = Butter{hiB[0], hiB[1], hiB[2], hiA[1], hiA[2]};
        a.cur_low = cur_low[(size_t)i];
        a.ops = io.ops;
        dim3 grid(cdiv(a.l.w, RT_W), cdiv(a.l.h, RT_H), lanes);
        KLAUNCH("riesz_phase", i, k_riesz_phase<<<grid, 256, 0, ctx.stream>>>(a));
    }
    // *old = *cur (before amplification, :267): the buffers just written become `old`
    for (int i = 0; i < nb; ++i) {
        std::swap(cur_low[(size_t)i], old_low[(size_t)i]);
        std::swap(cur_rx[(size_t)i], old_rx[(size_t)i]);
        std::swap(cur_ry[(size_t)i], old_ry[(size_t)i]);
    }
    if (ctx.opt.analysis_only) {   // state-carry pass of temporal sharding: pyramids and filter registers are up to date
        *produced = 0;
        return MC_OK;
    }
    if (plan.n_run == 0) return MC_OK;   // only first frames (passthrough) and held lanes
    // this frame's band/pair now live in the old_* buffers
    for (int i = nb - 1; i >= 0; --i)
        MCK_ST(amplify(ctx, p, i, lanes, io.ops, amp[(size_t)i], t_c[(size_t)i], t_s[(size_t)i], old_low[(size_t)i], old_rx[(size_t)i],
                       old_ry[(size_t)i], low_amp[(size_t)i]));
    MCK_ST(collapse_egress(ctx, io, lab16, oct[(size_t)levels - 1], low_amp, res, tm_band, tm_valid, ctx.float_out));
    plan.produced(ctx, true, false, produced);
    return MC_OK;
}

// A clip as `frames` frame calls: frame 0 with the handle's ops, every later frame RUN for the lanes that are not held.
mc_status RieszMode::frame_loop(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int nlevels, int* produced, int frames) {
    std::vector<uint8_t> later(ctx.lane_ops, ctx.lane_ops + lanes);
    for (uint8_t& o : later)
        if (o != LANE_HOLD) o = LANE_RUN;
    for (int t = 0; t < frames; ++t) {
        ModeCtx c = ctx;
        if (t > 0) c.lane_ops = later.data();
        c.lane_produced = ctx.lane_produced + (size_t)t * lanes;
        FrameIO f = io;
        f.in = io.in + (size_t)t * lanes * io.in_lane_stride;
        f.out = io.out + (size_t)t * lanes * io.out_lane_stride;
        int any = 0;
        MCK_ST(process(c, f, p, nlevels, &any));
        *produced |= any;
    }
    lab16_frame = false;   // a clip call, even one run as frame calls
    return MC_OK;
}

// One clip: the launch set of a frame call over V = frames * lanes virtual lanes, with the phase kernel replaced by
// k_riesz_phase_clip (state in registers across the clip).  The result is that of `frames` frame calls.
mc_status RieszMode::run_clip(const ModeCtx& ctx, const FrameIO& io0, const mc_params& p, int frames, bool first, int* produced) {
    const int vl = frames * lanes, nb = levels - 1;
    MCK_ST(ClipScratch::grow(clip, ctx, vl, (size_t)vl * 3 * plane16 * sizeof(int16_t), (size_t)w * h * 3, [&]() -> mc_status {
        const size_t v = (size_t)vl;
        clip.oct.assign((size_t)levels, nullptr);
        clip.band.assign((size_t)levels, nullptr);
        clip.rx.assign((size_t)levels, nullptr);
        clip.ry.assign((size_t)levels, nullptr);
        clip.tm_oct.assign((size_t)levels, TensorMapStorage{});
        clip.tm_band.assign((size_t)levels, TensorMapStorage{});
        clip.tm_amp.assign((size_t)levels, TensorMapStorage{});
        clip.tm_valid.assign((size_t)levels, 0);
        for (int i = 0; i < levels; ++i) {
            const Level& l = lv[(size_t)i];
            MCK(clip.arena.alloc(&clip.oct[(size_t)i], v * l.plane));
            if (i >= nb) continue;
            MCK(clip.arena.alloc(&clip.band[(size_t)i], v * l.plane));
            MCK(clip.arena.alloc(&clip.rx[(size_t)i], v * l.plane));
            MCK(clip.arena.alloc(&clip.ry[(size_t)i], v * l.plane));
            clip.tm_valid[(size_t)i] = make_tensor_map_box(&clip.tm_oct[(size_t)i], clip.oct[(size_t)i], l, vl, R9_SW, R9_SH) &&
                                       make_tensor_map_box(&clip.tm_band[(size_t)i], clip.band[(size_t)i], l, vl, RT_SW, RT_SH) &&
                                       make_tensor_map_box(&clip.tm_amp[(size_t)i], clip.rx[(size_t)i], l, vl, R9_SW, R9_SH) ? 1 : 0;
        }
        if (nb > 0) {
            MCK(clip.arena.alloc(&clip.amp, v * lv[0].plane));
            MCK(clip.arena.alloc(&clip.t_c, v * lv[0].plane));
            MCK(clip.arena.alloc(&clip.t_s, v * lv[0].plane));
        }
        return MC_OK;
    }));
    bool rebuild_old = false;
    if (!first) MCK_ST(apply_cutoffs(ctx, p, &rebuild_old));
    const uint8_t* ops0 = nullptr;   // per-lane ops of the clip's first frame (null when uniform)
    MCK(plan.upload(ctx, &ops0));
    FrameIO io = io0;   // every frame of every lane
    io.lanes = vl;
    MCK(clip.upload_vops(ctx, plan, frames, plan.n_run != lanes, &io.ops));
    MCK_ST(build_pyramid(ctx, io, clip.lab16, clip.oct, clip.band, clip.tm_oct, clip.tm_valid));
    // per band level: the temporal loop, then the amplification of every frame (its amp / t_c / t_s scratch is reused
    // by the next level)
    for (int i = nb - 1; i >= 0; --i) {
        PhaseClipArgs a;
        a.l = lv[(size_t)i];
        a.band = clip.band[(size_t)i];
        a.rx = ctx.opt.analysis_only ? nullptr : clip.rx[(size_t)i];
        a.ry = ctx.opt.analysis_only ? nullptr : clip.ry[(size_t)i];
        a.amp = ctx.opt.analysis_only ? nullptr : clip.amp;
        a.t_c = ctx.opt.analysis_only ? nullptr : clip.t_c;
        a.t_s = ctx.opt.analysis_only ? nullptr : clip.t_s;
        a.old_low = old_low[(size_t)i]; a.old_rx = old_rx[(size_t)i]; a.old_ry = old_ry[(size_t)i];
        a.ph_c = phase_c[(size_t)i]; a.ph_s = phase_s[(size_t)i];
        a.lo_r0c = lo_r0c[(size_t)i]; a.lo_r0s = lo_r0s[(size_t)i]; a.lo_r1c = lo_r1c[(size_t)i]; a.lo_r1s = lo_r1s[(size_t)i];
        a.hi_r0c = hi_r0c[(size_t)i]; a.hi_r0s = hi_r0s[(size_t)i]; a.hi_r1c = hi_r1c[(size_t)i]; a.hi_r1s = hi_r1s[(size_t)i];
        a.lo = Butter{loB[0], loB[1], loB[2], loA[1], loA[2]};
        a.hi = Butter{hiB[0], hiB[1], hiB[2], hiA[1], hiA[2]};
        a.first = first ? 1 : 0;
        a.rebuild_old = rebuild_old ? 1 : 0;
        a.ops = ops0;
        dim3 grid(cdiv(a.l.w, RT_W), cdiv(a.l.h, RT_H), lanes);
        const CUtensorMap& tm = *reinterpret_cast<const CUtensorMap*>(&clip.tm_band[(size_t)i]);
        if (ctx.opt.use_tma && clip.tm_valid[(size_t)i])
            KLAUNCH("riesz_phase_clip", i, k_riesz_phase_clip<true><<<grid, 256, 0, ctx.stream>>>(a, frames, lanes, tm));
        else
            KLAUNCH("riesz_phase_clip", i, k_riesz_phase_clip<false><<<grid, 256, 0, ctx.stream>>>(a, frames, lanes, tm));
        if (ctx.opt.analysis_only) continue;
        // the amplified band overwrites the Riesz pair's rx, point for point
        MCK_ST(amplify(ctx, p, i, vl, io.ops, clip.amp, clip.t_c, clip.t_s, clip.band[(size_t)i], clip.rx[(size_t)i], clip.ry[(size_t)i],
                       clip.rx[(size_t)i]));
    }
    if (ctx.opt.analysis_only) return MC_OK;   // state-carry pass: nothing is produced
    // level i's collapse result overwrites its band, which amplify was the last to read
    MCK_ST(collapse_egress(ctx, io, clip.lab16, clip.oct[(size_t)levels - 1], clip.rx, clip.band, clip.tm_amp, clip.tm_valid,
                           ctx.float_out ? clip.fout : nullptr));
    MCK_ST(clip.copy_last_tap(ctx, plan, frames, (size_t)w * h * 3));
    // frame 0 as a frame call (first frames pass through); every later frame is RUN for the lanes that are not held
    plan.produced(ctx, true, false, produced, frames, true);
    return MC_OK;
}

void RieszMode::find_state(const char* name, int level, StateRef& out) {
    out = StateRef{};
    if (!std::strcmp(name, "lab16")) {   // before the band-level guard: a 1-level pyramid has no band level
        if (level == 0) lab16_state(lab16, lab16_frame, w, h, pitch16, plane16, out);
        return;
    }
    if (!allocated || level < 0 || level >= levels - 1) return;
    struct { const char* n; std::vector<float*>* v; } map[] = {
        {"old.lowpass", &old_low}, {"old.rx", &old_rx}, {"old.ry", &old_ry}, {"phase.c", &phase_c}, {"phase.s", &phase_s},
        {"lo.r0.c", &lo_r0c}, {"lo.r0.s", &lo_r0s}, {"lo.r1.c", &lo_r1c}, {"lo.r1.s", &lo_r1s},
        {"hi.r0.c", &hi_r0c}, {"hi.r0.s", &hi_r0s}, {"hi.r1.c", &hi_r1c}, {"hi.r1.s", &hi_r1s}};
    for (auto& m : map)
        if (!std::strcmp(name, m.n)) {
            const Level& l = lv[(size_t)level];
            out.ptr = (*m.v)[(size_t)level]; out.rows = l.h; out.cols = l.w; out.channels = 1; out.pitch = l.pitch; out.plane_stride = l.plane;
            return;
        }
}

}  // namespace mc
