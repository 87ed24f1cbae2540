// Front of the reference chain fused onto the device (SURVEY.md 8f-1): PreprocessProcessor (normalised ROI crop +
// INTER_AREA 1/2..1/8 downscale, reference src/processing/PreprocessProcessor.cpp:10-51) and GrayscaleProcessor
// (BGR2GRAY, src/processing/GrayscaleProcessor.cpp:7-16), bit-exact with OpenCV's u8 paths (mc_math.cuh), in one kernel
// over every virtual lane whose source is u8 BGR, u8 gray or NV12 planes (an NV12 pixel is converted as
// cvtColor(YUV2BGR_NV12) converts it inside the tap walk, so no full-resolution BGR frame is ever stored); and the NV12
// conversions around the magnifier for the video decoder / encoder hand-off.
#include "mc_internal.h"

namespace mc {

namespace {

// Source pixels as the front kernel reads them: (sx, sy) relative to the ROI origin (ox, oy) of virtual lane v.
template <int SRC> struct FrontPx;
template <> struct FrontPx<FRONT_BGR> {
    const uint8_t* p; size_t step;
    __device__ void operator()(int sx, int sy, int (&v)[3]) const {
        const uint8_t* q = p + (size_t)sy * step + (size_t)3 * sx;
        v[0] = __ldg(q); v[1] = __ldg(q + 1); v[2] = __ldg(q + 2);
    }
};
template <> struct FrontPx<FRONT_GRAY> {
    const uint8_t* p; size_t step;
    __device__ void operator()(int sx, int sy, int (&v)[1]) const { v[0] = __ldg(p + (size_t)sy * step + sx); }
};
template <> struct FrontPx<FRONT_NV12> {   // cvtColor(YUV2BGR_NV12) of the pixel: its luma and its 2x2 block's Cb,Cr
    const uint8_t* y; const uint8_t* uv; size_t pitch; int ox, oy;
    __device__ void operator()(int sx, int sy, int (&v)[3]) const {
        const int ax = ox + sx, ay = oy + sy;
        const uint8_t* c = uv + (size_t)(ay >> 1) * pitch + (ax & ~1);
        uint8_t b, g, r;
        nv12_to_bgr_px(__ldg(y + (size_t)ay * pitch + ax), __ldg(c), __ldg(c + 1), b, g, r);
        v[0] = b; v[1] = g; v[2] = r;
    }
};

// One thread per output pixel of one virtual lane (blockIdx.z): every channel of the preprocessed pixel and its gray
// byte from one walk over the pixel's source taps.
template <int SRC>
__global__ void __launch_bounds__(256) k_chain_front(const FrontArgs a) {
    constexpr int CN = SRC == FRONT_GRAY ? 1 : 3;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const size_t v = blockIdx.z;
    if (x >= a.dw || (a.flags && !a.flags[v])) return;
    FrontPx<SRC> px;
    if constexpr (SRC == FRONT_NV12) {
        px = FrontPx<SRC>{a.src + v * a.lane_stride, a.uv + v * a.lane_stride, a.step, a.rx, a.ry};
    } else {
        px = FrontPx<SRC>{a.src + v * a.lane_stride + (size_t)a.ry * a.step + (size_t)CN * a.rx, a.step};
    }
    int o[CN];
    if (a.kind == FRONT_COPY) px(x, y, o);
    else resize_area_px<CN>(px, y, x, a.isx, a.isy, a.kind == FRONT_AREA_FAST, a.xtab, a.xofs, a.ytab, a.yofs, o);
    if (a.dst) {
        uint8_t* d = a.dst + v * a.dst_lane_stride + (size_t)y * a.dst_step + (size_t)CN * x;
#pragma unroll
        for (int c = 0; c < CN; ++c) d[c] = (uint8_t)o[c];
    }
    if constexpr (CN == 3) {
        if (a.gray) a.gray[(v * a.dh + y) * a.dw + x] = bgr_to_gray_u8(o[0], o[1], o[2]);
    }
}

}  // namespace

cudaError_t launch_chain_front(const FrontArgs& a, int src, int vlanes, cudaStream_t s) {
    const dim3 grid((unsigned)((a.dw + 255) / 256), (unsigned)a.dh, (unsigned)vlanes);
    switch (src) {
        case FRONT_BGR: k_chain_front<FRONT_BGR><<<grid, 256, 0, s>>>(a); break;
        case FRONT_GRAY: k_chain_front<FRONT_GRAY><<<grid, 256, 0, s>>>(a); break;
        default: k_chain_front<FRONT_NV12><<<grid, 256, 0, s>>>(a); break;
    }
    return cudaGetLastError();
}

// ---- NV12 frames in and out of the magnifier (the hand-off format of hardware video decoders and encoders): the
// conversions to and from the packed BGR frames the modes work on, bit-exact with OpenCV's u8 fixed point
// (nv12_to_bgr_px / bgr_to_ycc_px in mc_math.cuh).  Both kernels are bandwidth-bound: 1.5 B/px of NV12 and 3 B/px of
// BGR per pixel.  A thread owns a 2-row x 8-column block: one 64-bit load or store per luma row, one for the 4 Cb,Cr
// pairs of the block, and three per BGR row (24 bytes); rows or pointers that are not 8-byte aligned, and the last
// columns of a row whose width is not a multiple of 8, take the byte path.

namespace {

constexpr int kBlockX = 32, kBlockY = 4;   // threads: 32 column groups of 8 x 4 row pairs

struct ToBgrArgs {
    const uint8_t* y;
    const uint8_t* uv;
    size_t pitch, lane_stride;
    uint8_t* bgr;
    size_t bgr_step;
    int w, h;
    int vec_in, vec_out;   // the NV12 planes / the BGR rows allow 64-bit accesses
};

struct ToNv12Args {
    const uint8_t* bgr;
    size_t bgr_step;
    uint8_t* y;
    uint8_t* uv;
    size_t pitch, lane_stride;
    int w, h;
    int vec_in, vec_out;   // the BGR rows / the NV12 planes allow 64-bit accesses
    const uint8_t* flags;  // one byte per lane, or null: every lane
};

__device__ __forceinline__ void load8(const uint8_t* __restrict__ p, bool vec, int n, uint8_t (&v)[8]) {
    if (vec) {
        const uint2 q = __ldg(reinterpret_cast<const uint2*>(p));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            v[i] = (uint8_t)(q.x >> (8 * i));
            v[4 + i] = (uint8_t)(q.y >> (8 * i));
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = i < n ? __ldg(p + i) : (uint8_t)0;
    }
}

template <int N>
__device__ __forceinline__ void store(uint8_t* __restrict__ p, bool vec, int n, const uint8_t (&v)[N]) {
    if (vec) {
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            uint2 q;
            q.x = (unsigned)v[8 * j] | (unsigned)v[8 * j + 1] << 8 | (unsigned)v[8 * j + 2] << 16 | (unsigned)v[8 * j + 3] << 24;
            q.y = (unsigned)v[8 * j + 4] | (unsigned)v[8 * j + 5] << 8 | (unsigned)v[8 * j + 6] << 16 | (unsigned)v[8 * j + 7] << 24;
            reinterpret_cast<uint2*>(p)[j] = q;
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i)
            if (i < n) p[i] = v[i];
    }
}

__global__ void __launch_bounds__(kBlockX * kBlockY) k_nv12_to_bgr(const ToBgrArgs a) {
    const int x0 = (blockIdx.x * kBlockX + threadIdx.x) * 8;
    const int r = blockIdx.y * kBlockY + threadIdx.y;   // row pair
    if (x0 >= a.w || 2 * r >= a.h) return;
    const size_t lane = blockIdx.z;
    const int n = min(8, a.w - x0);                     // even: w is
    const bool full = n == 8;
    const uint8_t* yp = a.y + lane * a.lane_stride + (size_t)(2 * r) * a.pitch + x0;
    uint8_t y0[8], y1[8], c[8];
    load8(yp, full && a.vec_in, n, y0);
    load8(yp + a.pitch, full && a.vec_in, n, y1);
    load8(a.uv + lane * a.lane_stride + (size_t)r * a.pitch + x0, full && a.vec_in, n, c);
    uint8_t o0[24], o1[24];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int u = c[i & ~1], v = c[i | 1];
        nv12_to_bgr_px(y0[i], u, v, o0[3 * i], o0[3 * i + 1], o0[3 * i + 2]);
        nv12_to_bgr_px(y1[i], u, v, o1[3 * i], o1[3 * i + 1], o1[3 * i + 2]);
    }
    uint8_t* op = a.bgr + lane * a.bgr_step * a.h + (size_t)(2 * r) * a.bgr_step + (size_t)3 * x0;
    store(op, full && a.vec_out, 3 * n, o0);
    store(op + a.bgr_step, full && a.vec_out, 3 * n, o1);
}

__global__ void __launch_bounds__(kBlockX * kBlockY) k_bgr_to_nv12(const ToNv12Args a) {
    const size_t lane = blockIdx.z;
    if (a.flags && !a.flags[lane]) return;
    const int x0 = (blockIdx.x * kBlockX + threadIdx.x) * 8;
    const int r = blockIdx.y * kBlockY + threadIdx.y;
    if (x0 >= a.w || 2 * r >= a.h) return;
    const int n = min(8, a.w - x0);
    const bool full = n == 8;
    const uint8_t* ip = a.bgr + lane * a.bgr_step * a.h + (size_t)(2 * r) * a.bgr_step + (size_t)3 * x0;
    uint8_t i0[24], i1[24];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        uint8_t t0[8], t1[8];
        const int nk = min(8, max(0, 3 * n - 8 * k));
        load8(ip + 8 * k, full && a.vec_in, nk, t0);
        load8(ip + a.bgr_step + 8 * k, full && a.vec_in, nk, t1);
#pragma unroll
        for (int i = 0; i < 8; ++i) { i0[8 * k + i] = t0[i]; i1[8 * k + i] = t1[i]; }
    }
    uint8_t y0[8], y1[8], c[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint8_t cb, cr, cb1, cr1;
        bgr_to_ycc_px(i0[3 * i], i0[3 * i + 1], i0[3 * i + 2], y0[i], cb, cr);
        bgr_to_ycc_px(i1[3 * i], i1[3 * i + 1], i1[3 * i + 2], y1[i], cb1, cr1);   // chroma unused: dead code
        if ((i & 1) == 0) { c[i] = cb; c[i + 1] = cr; }
    }
    uint8_t* yp = a.y + lane * a.lane_stride + (size_t)(2 * r) * a.pitch + x0;
    store(yp, full && a.vec_out, n, y0);
    store(yp + a.pitch, full && a.vec_out, n, y1);
    store(a.uv + lane * a.lane_stride + (size_t)r * a.pitch + x0, full && a.vec_out, n, c);
}

bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

dim3 grid_of(int w, int h, int lanes) {
    const int groups = (w + 7) / 8;
    return dim3((unsigned)((groups + kBlockX - 1) / kBlockX), (unsigned)((h / 2 + kBlockY - 1) / kBlockY), (unsigned)lanes);
}

}  // namespace

cudaError_t launch_nv12_to_bgr(const Nv12Planes& in, int w, int h, int lanes, uint8_t* bgr, size_t bgr_step, cudaStream_t s) {
    ToBgrArgs a;
    a.y = in.y; a.uv = in.uv; a.pitch = in.pitch; a.lane_stride = in.lane_stride;
    a.bgr = bgr; a.bgr_step = bgr_step; a.w = w; a.h = h;
    a.vec_in = aligned8(in.y) && aligned8(in.uv) && in.pitch % 8 == 0 && (lanes == 1 || in.lane_stride % 8 == 0);
    a.vec_out = aligned8(bgr) && bgr_step % 8 == 0;
    k_nv12_to_bgr<<<grid_of(w, h, lanes), dim3(kBlockX, kBlockY), 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_bgr_to_nv12(const uint8_t* bgr, size_t bgr_step, int w, int h, int lanes, const uint8_t* flags,
                               uint8_t* y, uint8_t* uv, size_t pitch, size_t lane_stride, cudaStream_t s) {
    ToNv12Args a;
    a.bgr = bgr; a.bgr_step = bgr_step; a.y = y; a.uv = uv; a.pitch = pitch; a.lane_stride = lane_stride;
    a.w = w; a.h = h; a.flags = flags;
    a.vec_in = aligned8(bgr) && bgr_step % 8 == 0;
    a.vec_out = aligned8(y) && aligned8(uv) && pitch % 8 == 0 && (lanes == 1 || lane_stride % 8 == 0);
    k_bgr_to_nv12<<<grid_of(w, h, lanes), dim3(kBlockX, kBlockY), 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace mc
