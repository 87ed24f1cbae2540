// Front of the reference chain fused onto the device (SURVEY.md 8f-1): PreprocessProcessor (normalised ROI crop +
// INTER_AREA 1/2..1/8 downscale, reference src/processing/PreprocessProcessor.cpp:10-51) and GrayscaleProcessor
// (BGR2GRAY, src/processing/GrayscaleProcessor.cpp:7-16), bit-exact with OpenCV's u8 paths (mc_math.cuh), in one kernel
// over every virtual lane whose source is u8 BGR, u8 gray, 4:2:0 planes (NV12 or I420 / YV12) or a packed 4:2:2 camera
// frame (YUYV / UYVY; a 4:2:0 or 4:2:2 pixel is converted as cvtColor converts it inside the tap walk, so no
// full-resolution BGR frame needs to be stored); and the NV12
// conversions around the magnifier for the video decoder / encoder hand-off, and the export canvas built from the chain's
// two taps (the exporter's compose, SURVEY.md 8f-2).
#include "../../include/magcore_b200.h"
#include "mc_internal.h"

namespace mc {

namespace {

// Source pixels as the front kernel reads them: (sx, sy) relative to the ROI origin (ox, oy) of virtual lane v.
template <int SRC> struct FrontPx;
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
// cvtColor(YUV2BGR_I420) of the pixel: the same arithmetic, its block's Cb and Cr from two planes `cpitch` bytes per row.
// The FRONT_NV12 instance walks its taps with this functor when the chroma is planar (FrontArgs::cstep), so the NV12 walk
// keeps the address arithmetic of an interleaved pair.
struct I420Px {
    const uint8_t* y; const uint8_t* u; const uint8_t* w; size_t pitch, cpitch; int ox, oy;
    __device__ void operator()(int sx, int sy, int (&v)[3]) const {
        const int ax = ox + sx, ay = oy + sy;
        const size_t c = (size_t)(ay >> 1) * cpitch + (ax >> 1);
        uint8_t b, g, r;
        nv12_to_bgr_px(__ldg(y + (size_t)ay * pitch + ax), __ldg(u + c), __ldg(w + c), b, g, r);
        v[0] = b; v[1] = g; v[2] = r;
    }
};
// cvtColor(YUV2BGR_YUYV / _UYVY) of the pixel: its Y and its group's Cb,Cr, the group read as one 32-bit word when every
// group is 4-byte aligned (vec), else byte by byte.  p is the ROI's first row; the group of a pixel follows from its
// column in the frame (ox + sx), so a crop at an odd column still pairs the frame's pixels.
template <bool UYVY> struct Yuv422Px {
    const uint8_t* p; size_t pitch; int ox; bool vec;
    __device__ void operator()(int sx, int sy, int (&v)[3]) const {
        const int ax = ox + sx;
        const uint8_t* q = p + (size_t)sy * pitch + (size_t)2 * (ax & ~1);
        const uint32_t grp = vec ? __ldg(reinterpret_cast<const unsigned*>(q))
                                 : (uint32_t)__ldg(q) | (uint32_t)__ldg(q + 1) << 8 | (uint32_t)__ldg(q + 2) << 16 |
                                       (uint32_t)__ldg(q + 3) << 24;
        uint8_t b, g, r;
        yuv422_to_bgr_px(grp, ax & 1, UYVY, b, g, r);
        v[0] = b; v[1] = g; v[2] = r;
    }
};
template <> struct FrontPx<FRONT_YUYV> : Yuv422Px<false> {};
template <> struct FrontPx<FRONT_UYVY> : Yuv422Px<true> {};
// A BGR pixel, or COLOR_RGB2BGR / RGBA2BGR / BGRA2BGR (planar: a merge of the B, G, R planes) of an RGB one: its three
// channel bytes at b / g / r + sy * pitch + sx * pstep, the bases already at the ROI origin.  One functor serves BGR and
// all four RGB layouts.
struct RgbPx {
    const uint8_t* b; const uint8_t* g; const uint8_t* r; size_t pitch; int pstep;
    __device__ void operator()(int sx, int sy, int (&v)[3]) const {
        const size_t o = (size_t)sy * pitch + (size_t)sx * pstep;
        v[0] = __ldg(b + o); v[1] = __ldg(g + o); v[2] = __ldg(r + o);
    }
};

// The preprocessed pixel (x, y): its ROI tap, or its INTER_AREA taps, read through px.
template <int CN, class Px>
__device__ __forceinline__ void front_walk(const FrontArgs& a, const Px& px, int x, int y, int (&o)[CN]) {
    if (a.kind == FRONT_COPY) px(x, y, o);
    else resize_area_px<CN>(px, y, x, a.isx, a.isy, a.kind == FRONT_AREA_FAST, a.xtab, a.xofs, a.ytab, a.yofs, o);
}

// One thread per output pixel of one virtual lane (blockIdx.z): every channel of the preprocessed pixel and its gray
// byte from one walk over the pixel's source taps.  The per-lane origins cost registers: every instance but the BGR one
// is held to 32 (8 CTAs per SM, as before them) with no spills (-Xptxas -v).  The BGR instance spills under any bound
// and runs unbounded at 40, which allocates as the 34 it used before them did (6 CTAs per SM).
template <int SRC>
__global__ void __launch_bounds__(256, SRC == FRONT_BGR ? 0 : 8) k_chain_front(const FrontArgs a) {
    constexpr int CN = SRC == FRONT_GRAY ? 1 : 3;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const size_t v = blockIdx.z;
    if (x >= a.dw || (a.flags && !a.flags[v])) return;
    // the lane's crop origin: every lane's rectangle has the size dw x dh maps from, so the tap tables are shared
    const int2 org = a.org ? a.org[v] : make_int2(a.rx, a.ry);
    const int rx = org.x, ry = org.y;
    int o[CN];
    if constexpr (SRC == FRONT_NV12) {   // one uniform branch on the chroma layout
        const size_t l = v * a.lane_stride;
        if (a.cstep == kNv12ChromaStep) front_walk(a, FrontPx<SRC>{a.src + l, a.cb + l, a.step, rx, ry}, x, y, o);
        else front_walk(a, I420Px{a.src + l, a.cb + l, a.cr + l, a.step, a.cpitch, rx, ry}, x, y, o);
    } else if constexpr (SRC == FRONT_YUYV || SRC == FRONT_UYVY) {
        FrontPx<SRC> px;
        px.p = a.src + v * a.lane_stride + (size_t)ry * a.step; px.pitch = a.step; px.ox = rx; px.vec = a.vec != 0;
        front_walk(a, px, x, y, o);
    } else if constexpr (SRC == FRONT_BGR) {   // BGR and every RGB layout: three channel bases
        const size_t l = v * a.lane_stride + (size_t)ry * a.step + (size_t)rx * a.cstep;
        front_walk(a, RgbPx{a.src + l, a.cb + l, a.cr + l, a.step, a.cstep}, x, y, o);
    } else {
        front_walk(a, FrontPx<SRC>{a.src + v * a.lane_stride + (size_t)ry * a.step + (size_t)CN * rx, a.step}, x, y, o);
    }
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

cudaError_t launch_chain_front(const FrontArgs& args, int src, int vlanes, cudaStream_t s) {
    FrontArgs a = args;
    a.vec = (reinterpret_cast<uintptr_t>(a.src) & 3) == 0 && a.step % 4 == 0 && (vlanes == 1 || a.lane_stride % 4 == 0);
    const dim3 grid((unsigned)((a.dw + 255) / 256), (unsigned)a.dh, (unsigned)vlanes);
    switch (src) {
        case FRONT_BGR:   // the B, G, R channel bases of a BGR frame, the RGB family's fifth layout
            a.cb = a.src + 1; a.cr = a.src + 2; a.cstep = 3;
            [[fallthrough]];
        case FRONT_RGB: k_chain_front<FRONT_BGR><<<grid, 256, 0, s>>>(a); break;
        case FRONT_GRAY: k_chain_front<FRONT_GRAY><<<grid, 256, 0, s>>>(a); break;
        case FRONT_YUYV: k_chain_front<FRONT_YUYV><<<grid, 256, 0, s>>>(a); break;
        case FRONT_UYVY: k_chain_front<FRONT_UYVY><<<grid, 256, 0, s>>>(a); break;
        default: k_chain_front<FRONT_NV12><<<grid, 256, 0, s>>>(a); break;
    }
    return cudaGetLastError();
}

// ---- NV12 frames in and out of the magnifier (the hand-off format of hardware video decoders and encoders): the
// conversions to and from the packed BGR frames the modes work on, bit-exact with OpenCV's u8 fixed point
// (nv12_to_bgr_px / bgr_to_ycc_px in mc_math.cuh); and the export canvas of Exporter.cpp:25-34, 53-88 (labels as the
// handle's overlay of per-pixel tone maps),
// whose panes are BGR, gray (GRAY2BGR), 4:2:0 or 4:2:2 sources and whose canvas is BGR, NV12 or I420.  All three kernels
// are bandwidth-bound: 1.5 B/px of 4:2:0 and 3 B/px of BGR per pixel.  A thread owns a 2-row x 8-column block: one 64-bit
// load or store per luma or gray row, one for the 4 Cb,Cr pairs of the block (I420: one 32-bit access per chroma plane),
// and three per BGR row (24 bytes); rows or pointers that are not 8-byte aligned (I420 chroma: 4-byte), a canvas block
// that does not start on an 8-byte boundary, and the last columns of a row whose width is not a multiple of 8, take the
// byte path.  NV12 and I420 differ only in the chroma addressing (FrontArgs in mc_internal.h), one uniform branch.  The compose kernel with one BGR pane does
// k_bgr_to_nv12's job, but measured 3.64 against 3.45 us per 1080p frame on an H100 (tools/bench_nv12.py), so the NV12
// egress keeps its own kernel.

namespace {

constexpr int kBlockX = 32, kBlockY = 4;   // threads: 32 column groups of 8 x 4 row pairs

struct ToBgrArgs {
    Nv12Planes in;
    uint8_t* bgr;
    size_t bgr_step;
    int w, h;
    int vec_in, vec_out;   // the 4:2:0 planes / the BGR rows allow 64-bit (I420 chroma: 32-bit) accesses
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

__device__ __forceinline__ void load4(const uint8_t* __restrict__ p, bool vec, int n, uint8_t (&v)[4]) {
    if (vec) {
        const unsigned q = __ldg(reinterpret_cast<const unsigned*>(p));
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = (uint8_t)(q >> (8 * i));
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = i < n ? __ldg(p + i) : (uint8_t)0;
    }
}

// The Cb (u) and Cr (w) of the n / 2 2x2 blocks from column x0 (even) in chroma row r of a 4:2:0 frame's lane: one 64-bit
// load of the interleaved pairs (NV12) or one 32-bit load per plane (I420).
__device__ __forceinline__ void load_chroma(const uint8_t* cb, const uint8_t* cr, size_t cpitch, int cstep, bool vec, int x0,
                                            int r, int n, uint8_t (&u)[4], uint8_t (&w)[4]) {
    const size_t o = (size_t)r * cpitch + (size_t)(x0 >> 1) * cstep;
    if (cstep == kNv12ChromaStep) {
        uint8_t c[8];
        load8(cb + o, vec, n, c);
#pragma unroll
        for (int i = 0; i < 4; ++i) { u[i] = c[2 * i]; w[i] = c[2 * i + 1]; }
    } else {
        load4(cb + o, vec, n / 2, u);
        load4(cr + o, vec, n / 2, w);
    }
}

template <int N>
__device__ __forceinline__ void store(uint8_t* __restrict__ p, bool vec, int n, const uint8_t (&v)[N]) {
    if (vec && N == 4) {   // one 32-bit store (an I420 chroma row of a block)
        *reinterpret_cast<unsigned*>(p) = (unsigned)v[0] | (unsigned)v[1] << 8 | (unsigned)v[2] << 16 | (unsigned)v[3] << 24;
    } else if (vec) {
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
    const Nv12Planes& in = a.in;
    const uint8_t* yp = in.y + lane * in.lane_stride + (size_t)(2 * r) * in.pitch + x0;
    uint8_t y0[8], y1[8], cu[4], cv[4];
    load8(yp, full && a.vec_in, n, y0);
    load8(yp + in.pitch, full && a.vec_in, n, y1);
    load_chroma(in.cb + lane * in.lane_stride, in.cr + lane * in.lane_stride, in.cpitch, in.cstep, full && a.vec_in, x0, r, n,
                cu, cv);
    uint8_t o0[24], o1[24];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int u = cu[i >> 1], v = cv[i >> 1];
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
// Two rows (2r, 2r + 1) of n <= 8 pixels from column x0 of virtual lane v's frame in a pane source, as BGR bytes: gray
// expanded as GRAY2BGR, NV12 / I420 and YUYV / UYVY converted as cvtColor does (x0 and n are even, so the Cb,Cr pairs and
// the 4:2:2 groups are whole).
__device__ __forceinline__ void load_pane(const PaneSrc& s, bool vec, size_t v, int x0, int r, int n, uint8_t (&o0)[24],
                                          uint8_t (&o1)[24]) {
    const uint8_t* row = s.p + v * s.lane_stride + (size_t)(2 * r) * s.step;
    if (s.kind == FRONT_NV12) {
        uint8_t y0[8], y1[8], cu[4], cv[4];
        load8(row + x0, vec, n, y0);
        load8(row + s.step + x0, vec, n, y1);
        load_chroma(s.cb + v * s.lane_stride, s.cr + v * s.lane_stride, s.cpitch, s.cstep, vec, x0, r, n, cu, cv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int u = cu[i >> 1], w = cv[i >> 1];
            nv12_to_bgr_px(y0[i], u, w, o0[3 * i], o0[3 * i + 1], o0[3 * i + 2]);
            nv12_to_bgr_px(y1[i], u, w, o1[3 * i], o1[3 * i + 1], o1[3 * i + 2]);
        }
    } else if (s.kind == FRONT_YUYV || s.kind == FRONT_UYVY) {   // 4 groups of 4 bytes per row, from byte 2 * x0
        const bool uyvy = s.kind == FRONT_UYVY;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            uint8_t t0[8], t1[8];
            const int nk = min(8, max(0, 2 * n - 8 * k));
            load8(row + (size_t)2 * x0 + 8 * k, vec, nk, t0);
            load8(row + s.step + (size_t)2 * x0 + 8 * k, vec, nk, t1);
#pragma unroll
            for (int i = 0; i < 4; ++i) {   // pixel 4k + i: group 2k + i / 2
                const int g = 4 * (i >> 1);
                const uint32_t g0 = (uint32_t)t0[g] | (uint32_t)t0[g + 1] << 8 | (uint32_t)t0[g + 2] << 16 | (uint32_t)t0[g + 3] << 24;
                const uint32_t g1 = (uint32_t)t1[g] | (uint32_t)t1[g + 1] << 8 | (uint32_t)t1[g + 2] << 16 | (uint32_t)t1[g + 3] << 24;
                const int px = 3 * (4 * k + i);
                yuv422_to_bgr_px(g0, i & 1, uyvy, o0[px], o0[px + 1], o0[px + 2]);
                yuv422_to_bgr_px(g1, i & 1, uyvy, o1[px], o1[px + 1], o1[px + 2]);
            }
        }
    } else if (s.kind == FRONT_GRAY) {
        uint8_t g0[8], g1[8];
        load8(row + x0, vec, n, g0);
        load8(row + s.step + x0, vec, n, g1);
#pragma unroll
        for (int i = 0; i < 24; ++i) { o0[i] = g0[i / 3]; o1[i] = g1[i / 3]; }
    } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            uint8_t t0[8], t1[8];
            const int nk = min(8, max(0, 3 * n - 8 * k));
            load8(row + (size_t)3 * x0 + 8 * k, vec, nk, t0);
            load8(row + s.step + (size_t)3 * x0 + 8 * k, vec, nk, t1);
#pragma unroll
            for (int i = 0; i < 8; ++i) { o0[8 * k + i] = t0[i]; o1[8 * k + i] = t1[i]; }
        }
    }
}

// The overlay on canvas row y, columns cx .. cx + 7 held in p (BGR): each pixel inside a rect becomes map[index][v] per
// channel.  One index load per labelled pixel, one palette byte per channel.  Columns past the pane's last one are
// mapped too when a rect covers them (their index is inside that rect's plane) but never stored.
__device__ __forceinline__ void overlay_row(const ComposeArgs& a, int cx, int y, uint8_t (&p)[24]) {
#pragma unroll
    for (int i = 0; i < kOverlayRects; ++i) {
        const OverlayRect& o = a.ov[i];
        const int dy = y - o.y;
        if (i >= a.ov_rects || (unsigned)dy >= (unsigned)o.h || cx + 8 <= o.x || o.x + o.w <= cx) continue;
        const uint16_t* row = o.index + (size_t)dy * o.w;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int dx = cx + k - o.x;
            if ((unsigned)dx < (unsigned)o.w) {
                const uint8_t* t = a.ov_map + (size_t)__ldg(row + dx) * 256;
#pragma unroll
                for (int c = 0; c < 3; ++c) p[3 * k + c] = __ldg(t + p[3 * k + c]);
            }
        }
    }
}

__device__ __forceinline__ void swap_rb(uint8_t (&p)[24]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint8_t t = p[3 * k];
        p[3 * k] = p[3 * k + 2];
        p[3 * k + 2] = t;
    }
}

// The R, G and B bytes of a canvas row's 8 BGR pixels p into the planes of a planar RGB canvas, `o` bytes from each base.
__device__ __forceinline__ void store_planes(const ComposeArgs& a, size_t o, bool vec, int n, const uint8_t (&p)[24]) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        uint8_t q[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) q[k] = p[3 * k + 2 - c];
        store((c == 0 ? a.data : c == 1 ? a.uv : a.cr) + o, vec, n, q);
    }
}

// Whether the canvas box [x0, x0 + w) x [y0, y0 + h) meets a rect of the overlay.
__device__ __forceinline__ bool overlay_meets(const ComposeArgs& a, int x0, int y0, int w, int h) {
    bool hit = false;
#pragma unroll
    for (int i = 0; i < kOverlayRects; ++i) {
        const OverlayRect& o = a.ov[i];
        hit |= i < a.ov_rects && o.x < x0 + w && x0 < o.x + o.w && o.y < y0 + h && y0 < o.y + o.h;
    }
    return hit;
}

// One 2-row x 8-column block of one pane of virtual lane blockIdx.z's canvas.  blockIdx.y runs over the row blocks of
// pane 0, then those of pane 1, so a CTA stays inside one pane and reads one source.  A CTA whose canvas box meets an
// overlay rect maps its pixels in registers before they are stored or converted; the others take one uniform branch.
// Each row is mapped just before it is stored or converted, and 8 CTAs per SM (64 registers) keep the occupancy of the
// kernel without an overlay path, with no spills (-Xptxas -v).  OUT is the canvas format; MC_CANVAS_NV12 stands for both
// 4:2:0 canvases, NV12 and I420 (cr set).  The planar RGB canvas regathers both rows' bytes into three planes, which
// spills at 64 registers in every order tried (-Xptxas -v): its instance runs 6 CTAs per SM (80 registers) instead.
template <int OUT>
__global__ void __launch_bounds__(kBlockX * kBlockY, OUT == MC_CANVAS_RGB_PLANAR ? 6 : 8) k_compose(const ComposeArgs a) {
    const size_t v = blockIdx.z;
    const int op = a.ops ? a.ops[v] : COMPOSE_MAGNIFIED;
    if (op == COMPOSE_SKIP) return;
    const int pane = (int)blockIdx.y / a.pane_blocks;
    const int x0 = (blockIdx.x * kBlockX + threadIdx.x) * 8;
    const int r = ((int)blockIdx.y - pane * a.pane_blocks) * kBlockY + threadIdx.y;   // row pair of the pane
    if (x0 >= a.w || 2 * r >= a.h) return;
    const int i = a.split != MC_SPLIT_NONE && pane == 0 ? 0 : op == COMPOSE_FALLBACK ? 2 : 1;
    const PaneSrc s = i == 0 ? a.src[0] : i == 1 ? a.src[1] : a.src[2];
    const int n = min(8, a.w - x0);
    const bool full = n == 8;
    uint8_t p0[24], p1[24];
    load_pane(s, full && (a.vec_src >> i & 1), v, x0, r, n, p0, p1);
    const int cx = x0 + (a.split == MC_SPLIT_LEFT_RIGHT ? pane * a.w : 0);
    const int cy = 2 * r + (a.split == MC_SPLIT_TOP_BOTTOM ? pane * a.h : 0);
    const bool ov = a.ov_rects && overlay_meets(a, cx - 8 * (int)threadIdx.x, cy - 2 * (int)threadIdx.y, 8 * kBlockX, 2 * kBlockY);
    if (ov) overlay_row(a, cx, cy, p0);
    const bool vec = full && a.vec_out && cx % 8 == 0;
    uint8_t* row = a.data + v * a.lane_stride + (size_t)cy * a.pitch;
    if constexpr (OUT == MC_CANVAS_NV12) {
        uint8_t y0[8], y1[8], c[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            uint8_t cb, cr;
            bgr_to_ycc_px(p0[3 * k], p0[3 * k + 1], p0[3 * k + 2], y0[k], cb, cr);
            if ((k & 1) == 0) { c[k] = cb; c[k + 1] = cr; }
        }
        if (ov) overlay_row(a, cx, cy + 1, p1);   // row 0 is converted first: fewer bytes live while row 1 is mapped
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            uint8_t cb1, cr1;
            bgr_to_ycc_px(p1[3 * k], p1[3 * k + 1], p1[3 * k + 2], y1[k], cb1, cr1);   // chroma unused: dead code
        }
        store(row + cx, vec, n, y0);
        store(row + a.pitch + cx, vec, n, y1);
        if (a.cr) {   // I420: the block's 4 Cb and 4 Cr bytes into their planes, rows pitch / 2 apart
            uint8_t cu[4], cv[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) { cu[k] = c[2 * k]; cv[k] = c[2 * k + 1]; }
            const size_t o = v * a.lane_stride + (size_t)(cy / 2) * (a.pitch / 2) + cx / 2;
            store(a.uv + o, vec, n / 2, cu);
            store(a.cr + o, vec, n / 2, cv);
        } else {
            store(a.uv + v * a.lane_stride + (size_t)(cy / 2) * a.pitch + cx, vec, n, c);
        }
    } else if constexpr (OUT == MC_CANVAS_RGB_PLANAR) {   // one row store of n bytes per plane: R at data, G at uv, B at cr
        const size_t o = v * a.lane_stride + (size_t)cy * a.pitch + cx;
        store_planes(a, o, vec, n, p0);
        if (ov) overlay_row(a, cx, cy + 1, p1);
        store_planes(a, o + a.pitch, vec, n, p1);
    } else {   // BGR, or RGB: the BGR store with bytes 0 and 2 of each pixel exchanged
        if constexpr (OUT == MC_CANVAS_RGB) swap_rb(p0);
        store(row + (size_t)3 * cx, vec, 3 * n, p0);
        if (ov) overlay_row(a, cx, cy + 1, p1);
        if constexpr (OUT == MC_CANVAS_RGB) swap_rb(p1);
        store(row + a.pitch + (size_t)3 * cx, vec, 3 * n, p1);
    }
}

bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

// The chroma of a 4:2:0 frame allows the vector accesses of load_chroma / the compose kernel's chroma stores: 8-byte
// interleaved pairs (NV12; the luma checks cover the pitch) or 4-byte rows of both planes (I420).
bool chroma_vec(const uint8_t* cb, const uint8_t* cr, size_t cpitch, int cstep) {
    return cstep == kNv12ChromaStep ? aligned8(cb) : aligned4(cb) && aligned4(cr) && cpitch % 4 == 0;
}


dim3 grid_of(int w, int h, int lanes) {
    const int groups = (w + 7) / 8;
    return dim3((unsigned)((groups + kBlockX - 1) / kBlockX), (unsigned)((h / 2 + kBlockY - 1) / kBlockY), (unsigned)lanes);
}

}  // namespace

cudaError_t launch_nv12_to_bgr(const Nv12Planes& in, int w, int h, int lanes, uint8_t* bgr, size_t bgr_step, cudaStream_t s) {
    ToBgrArgs a;
    a.in = in;
    a.bgr = bgr; a.bgr_step = bgr_step; a.w = w; a.h = h;
    a.vec_in = aligned8(in.y) && chroma_vec(in.cb, in.cr, in.cpitch, in.cstep) && in.pitch % 8 == 0 &&
               (lanes == 1 || in.lane_stride % 8 == 0);
    a.vec_out = aligned8(bgr) && bgr_step % 8 == 0;
    k_nv12_to_bgr<<<grid_of(w, h, lanes), dim3(kBlockX, kBlockY), 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_compose(ComposeArgs a, int vlanes, cudaStream_t s) {
    const bool lane_vec = vlanes == 1;
    a.vec_src = 0;
    for (int i = 0; i < 3; ++i) {
        const PaneSrc& p = a.src[i];
        const bool vec = p.p && aligned8(p.p) && (p.kind != FRONT_NV12 || chroma_vec(p.cb, p.cr, p.cpitch, p.cstep)) &&
                         p.step % 8 == 0 && (lane_vec || p.lane_stride % 8 == 0);
        a.vec_src |= (int)vec << i;
    }
    const bool yuv420 = a.format == MC_CANVAS_NV12 || a.format == MC_CANVAS_I420;
    const bool planes_vec = yuv420 ? (a.cr ? aligned4(a.uv) && aligned4(a.cr) : aligned8(a.uv))
                                   : a.format != MC_CANVAS_RGB_PLANAR || (aligned8(a.uv) && aligned8(a.cr));
    a.vec_out = aligned8(a.data) && planes_vec && a.pitch % 8 == 0 && (lane_vec || a.lane_stride % 8 == 0);
    const int panes = a.split == MC_SPLIT_NONE ? 1 : 2;
    dim3 grid = grid_of(a.w, a.h, vlanes);
    a.pane_blocks = (int)grid.y;
    grid.y *= panes;
    const dim3 block(kBlockX, kBlockY);
    switch (a.format) {
        case MC_CANVAS_RGB: k_compose<MC_CANVAS_RGB><<<grid, block, 0, s>>>(a); break;
        case MC_CANVAS_RGB_PLANAR: k_compose<MC_CANVAS_RGB_PLANAR><<<grid, block, 0, s>>>(a); break;
        case MC_CANVAS_BGR: k_compose<MC_CANVAS_BGR><<<grid, block, 0, s>>>(a); break;
        default: k_compose<MC_CANVAS_NV12><<<grid, block, 0, s>>>(a); break;
    }
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
