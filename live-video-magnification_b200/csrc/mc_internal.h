// Internal interfaces between the handle (mc_core.cu), the tables (mc_tables.cpp) and the kernel
// launchers (mc_laplace.cu, mc_color.cu, mc_riesz.cu).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "mc_math.cuh"

namespace mc {

// Geometry of one pyramid level; planes are f32 [plane][h][pitch] with pitch % 32 == 0.
struct Level {
    int w = 0, h = 0, pitch = 0;
    size_t plane = 0;  // floats per plane = h * pitch
};

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

inline Level make_level(int w, int h) {
    Level l;
    l.w = w; l.h = h; l.pitch = round_up(w, 32); l.plane = (size_t)l.h * l.pitch;
    return l;
}

// Device constant tables shared by every handle on a device (built once per device).
struct DeviceTables {
    LabLutCell* lab_lut = nullptr;   // [34][33][33] cells (mc_math.cuh)
    LabLutPack* lab_pack = nullptr;  // the same cells packed into 16 B (mc_math.cuh)
    float4* inv_gamma = nullptr;      // [1024] spline coefficients {f, b, c, d}
    LabInvCoeffs inv_coeffs{};
};

// mc_tables.cpp ------------------------------------------------------------------------------
void build_lab_lut_cells(std::vector<LabLutCell>& out);          // from the embedded int16 table
void build_lab_lut_packs(const std::vector<LabLutCell>& cells, std::vector<LabLutPack>& out);   // empty if a field overflows
void build_inv_gamma_spline(std::vector<float4>& out);             // OpenCV sRGBInvGammaTab
void build_lab_inv_coeffs(LabInvCoeffs& out);
int calculate_max_levels(int w, int h);
int optimal_buffer_size(int fps);
void butterworth(unsigned order, double wn, std::vector<double>& a, std::vector<double>& b);
void motion_gains(double amplification, double coWavelength, int levels, int w, int h, std::vector<float>& gains);
void gaussian_kernel_13_3(float taps[13]);
void build_area_tab(int ssize, int dsize, double scale, std::vector<AreaTap>& tab, std::vector<int>& ofs);
void preprocess_roi(int cols, int rows, bool enabled, float rx, float ry, float rw, float rh, int& x, int& y, int& w, int& h);

// What one frame call does to one lane (stream) of a multi-lane handle.  The kernels read a per-frame device array of
// these, indexed by lane; a null array means every lane is RUN (the handle's uniform first frame is the `first` flag).
enum LaneOp : uint8_t {
    LANE_RUN = 0,     // the lane has temporal state: the ordinary frame
    LANE_FIRST = 1,   // the lane has no state: this frame is its first frame
    LANE_HOLD = 2,    // the lane is held: its state and its bytes of `out` are left untouched
};
__host__ __device__ __forceinline__ int lane_op(const uint8_t* ops, int lane) { return ops ? (int)ops[lane] : (int)LANE_RUN; }

// Calls f(a, b) once per run [a, b) of consecutive indices in [0, n) for which keep(i) holds, so that lanes (or frames)
// stored back to back move in one copy.  Stops at the first call that returns an error (non-zero) and returns it.
template <class Keep, class F>
auto for_each_run(size_t n, Keep keep, F f) -> decltype(f(n, n)) {
    for (size_t a = 0; a < n;) {
        if (!keep(a)) { ++a; continue; }
        size_t b = a;
        while (b < n && keep(b)) ++b;
        if (const auto r = f(a, b)) return r;
        a = b;
    }
    return {};
}

// ------------------------------------------------------------------------------------------------
// Laplace launchers (mc_laplace.cu).  All take the handle's stream; every call is one kernel launch
// and returns the launch's cudaError_t (cudaGetLastError()).
// ------------------------------------------------------------------------------------------------
struct FrameIO {
    const uint8_t* in = nullptr;   // [lanes][h][in_step]
    size_t in_step = 0, in_lane_stride = 0;
    uint8_t* out = nullptr;
    size_t out_step = 0, out_lane_stride = 0;
    int w = 0, h = 0, channels = 0, lanes = 0;
    const uint8_t* ops = nullptr;  // device LaneOp per lane of this FrameIO (already offset to its first lane) or null
};

// u8 BGR frame -> Lab int16 planes [lanes*3][h][pitch16] (exact OpenCV LUT values, SURVEY A.3)
// (l_f32 != null: also the L plane as f32 [lanes][h][l_pitch] — Phase's input)
cudaError_t launch_lab16(const FrameIO& io, const DeviceTables& tb, int16_t* lab, int pitch16, size_t plane16,
                         cudaStream_t s, float* l_f32 = nullptr, int l_pitch = 0, size_t l_plane = 0);

// fused ingest of the production path: u8 BGR -> Lab16 planes + G1 = pyrDown(Lab) (MagnifyCore.hpp:87-96, level 0)
cudaError_t launch_ingest_lab(const FrameIO& io, const DeviceTables& tb, int16_t* lab, int pitch16, size_t plane16,
                              float* g1, const Level& l1, cudaStream_t s);

struct LevelArgs {
    int in_kind = 0;           // 0: f32 planes, 1: Lab int16 planes, 2: u8 gray frame
    const void* g = nullptr;   // input planes of this level (fine)
    size_t in_plane = 0;       // elements between planes
    int in_row = 0;            // elements between rows
    int channels = 1;
    float sc[3] = {1, 1, 1}, of[3] = {0, 0, 0};   // value = fma(raw, sc[ch], of[ch]) for kinds 1, 2
    Level lf, lc;              // this level (fine) and the next (coarse)
    float* g_next = nullptr;   // G_{l+1} planes (written)
    float* hi = nullptr; float* lo = nullptr;     // state planes of this level
    float* m = nullptr;        // gain * (hi - lo), may be null
    int m_luma = 0;            // 1: m is stored for the L planes (channel 0) only: L-only synthesis reads no other
    int planes = 0;
    int first = 0;             // 1: hi = lo = band (MagnifyCore.hpp:98-103)
    int band = 1;              // 0: only pyrDown (the level-0 band never reaches the output)
    double c_hi = 0, one_minus_c_hi = 0, c_lo = 0, one_minus_c_lo = 0;
    float gain = 0;
    const void* tmap = nullptr;   // CUtensorMap of the f32 input planes (TMA-staged tile) or null
    const void* tmap_hi = nullptr, *tmap_lo = nullptr;   // CUtensorMaps of the state planes: prefetch their tiles too
    const uint8_t* ops = nullptr;   // device LaneOp per lane (plane / channels) or null: HOLD skips, FIRST acts as `first`
    // lanes whose parameters differ (mc_set_lane_params): per lane (plane / channels) {c_hi, 1 - c_hi, c_lo, 1 - c_lo} and
    // the gain, in place of the four coefficients and `gain` above; null: every lane uses those
    const double* lane_ema = nullptr;
    const float* lane_gain = nullptr;
};
// 128-byte opaque CUtensorMap storage + encoder for the level kernel's (72 x 39 x 1) box
struct alignas(64) TensorMapStorage { unsigned char bytes[128]; };
bool make_level_tensor_map(void* out_map, const float* base, const Level& l, int planes, bool state_tile = false);
// general form: box of box_w x box_h x 1 f32 elements (row bytes must be a multiple of 16)
bool make_tensor_map_box(void* out_map, const float* base, const Level& l, int planes, int box_w, int box_h);
// fused per level: pyrDown + pyrUp + subtract + dual-EMA update + gain (SpatialFilter.cpp:25-38,
// TemporalFilter.cpp:9-22, MagnifyCore.hpp:127-134)
cudaError_t launch_level(const LevelArgs& a, cudaStream_t s);
// the same over a clip of `frames` consecutive frames (mc_process_clip_device): the grid covers a.planes = lanes * C
// state planes, whose hi / lo tiles stay in registers for the whole clip.  Frame t of state plane p is virtual plane
// t * a.planes + p of the input (a.g, a.tmap over all virtual planes), a.g_next and a.m.  a.first / a.ops describe
// the clip's first frame; the later frames run.
cudaError_t launch_level_clip(const LevelArgs& a, int frames, cudaStream_t s);
// pure pyrDown of `a.g` into `a.g_next` (register/shuffle strip kernel; used when a.band == 0)
cudaError_t launch_down(const LevelArgs& a, cudaStream_t s);

// Where the synthesis kernels find a band: either a stored plane set (b == nullptr: value = a[i]) or the two
// temporal-filter state plane sets of that level, from which the amplified band-pass is rebuilt on the fly as
// gain * (a[i] - b[i]) = gain * (lowpassHi - lowpassLo) (TemporalFilter.cpp:21, MagnifyCore.hpp:127-134).
struct BandSrc {
    const float* a = nullptr;
    const float* b = nullptr;
    float gain = 1.0f;
    const float* lane_gain = nullptr;   // with b: the gain of each lane (mc_set_lane_params), in place of `gain`; or null
};

// out_l = pyrUp(coarse) + fine (SpatialFilter.cpp:52-61); `out` may be the stored fine plane itself (in place)
// over `planes` planes, the k-th being plane k * plane_stride of every source and of `out`
// (ops: device LaneOp per lane of `channels` planes, or null; HOLD lanes are skipped)
cudaError_t launch_collapse(const Level& lf, const Level& lc, const BandSrc& fine, const BandSrc& coarse, float* out, int planes,
                            cudaStream_t s, const uint8_t* ops = nullptr, int channels = 1, int plane_stride = 1);

// out = convert(input + chroma * pyrUp(pyrUp(c2) + m1)) (MagnifyCore.hpp:136-158).
// m1.a == nullptr: no motion; c2.a == nullptr: cur_1 = m1.  C == 3 reads `lab`, C == 1 reads io.in.
// io.ops: HOLD lanes are skipped, and with first_only also RUN lanes (analysis_only: only FIRST lanes are converted).
// luma_only (strip kernel, C == 3): only the L planes of m1 and c2 are read, a and b are the input's (a zero chroma
// factor; the caller guarantees that the a / b motion it skips is finite).
// lane_chroma (mc_set_lane_params): lane v's chroma is lane_chroma[v % chroma_lanes] in place of `chroma`; or null.
cudaError_t launch_egress(const FrameIO& io, const DeviceTables& tb, const int16_t* lab, int pitch16, size_t plane16,
                          const BandSrc& m1, const Level& l1, const BandSrc& c2, const Level& l2, float chroma,
                          float* float_out_or_null, cudaStream_t s, bool strip = true, bool first_only = false,
                          bool luma_only = false, const float* lane_chroma = nullptr, int chroma_lanes = 1);

// PreprocessProcessor + GrayscaleProcessor on the device (mc_preprocess.cu): one launch over `vlanes` virtual lanes.
// FRONT_YUYV + mc_yuv422_order is the packed 4:2:2 source of that byte order.  FRONT_NV12 is any 4:2:0 source, NV12 or
// I420 / YV12, told apart only by its chroma addressing (cb, cr, cpitch, cstep below).  FRONT_RGB is any RGB-family
// source (packed RGB, RGBA / BGRA, planar RGB): the B, G and R bytes of its pixel (x, y) are at src / cb / cr +
// y * step + x * cstep, cstep 3 or 4 for packed pixels and 1 for planes.  The front's FRONT_BGR instance walks every
// 3-channel packed or planar source this way, BGR itself with the bases src, src + 1, src + 2 and cstep 3.
enum FrontSrc { FRONT_BGR = 0, FRONT_GRAY = 1, FRONT_NV12 = 2, FRONT_YUYV = 3, FRONT_UYVY = 4, FRONT_RGB = 5 };
enum FrontKind { FRONT_COPY = 0, FRONT_AREA_FAST = 1, FRONT_AREA = 2 };   // crop only / integer INTER_AREA / general INTER_AREA
// The chroma of a 4:2:0 frame: the Cb and Cr of its 2x2 block (bx, by) are at cb[by * cpitch + bx * cstep] and
// cr[by * cpitch + bx * cstep].  NV12: cr = cb + 1, cstep 2, cpitch = the luma pitch; I420: two planes, cstep 1.
constexpr int kNv12ChromaStep = 2, kI420ChromaStep = 1;
struct FrontArgs {
    const uint8_t* src = nullptr;   // lane 0's frame (BGR / gray / YUYV / UYVY) or luma plane (4:2:0)
    const uint8_t* cb = nullptr;    // 4:2:0: lane 0's chroma, addressed as above
    const uint8_t* cr = nullptr;
    size_t cpitch = 0;
    int cstep = kNv12ChromaStep;
    size_t step = 0, lane_stride = 0;   // row pitch and virtual-lane stride of the source (the same for every plane)
    int rx = 0, ry = 0;             // ROI origin in the source
    const int2* org = nullptr;      // per virtual lane: its own ROI origin (mc_set_lane_roi) in place of rx / ry; or null
    int dw = 0, dh = 0;             // output size
    int kind = FRONT_COPY, isx = 1, isy = 1;
    const AreaTap* xtab = nullptr; const int* xofs = nullptr; const AreaTap* ytab = nullptr; const int* yofs = nullptr;
    uint8_t* dst = nullptr;         // preprocessed frames [v][dh][dst_step] (source channels), or null
    size_t dst_step = 0, dst_lane_stride = 0;
    uint8_t* gray = nullptr;        // their BGR2GRAY, tight [v][dh][dw], or null (3-channel sources only)
    const uint8_t* flags = nullptr; // per virtual lane, 0 = skip (held); null = every lane
    int vec = 0;                    // YUYV / UYVY: every group can be read as one 32-bit word (set by launch_chain_front)
};
cudaError_t launch_chain_front(const FrontArgs& a, int src, int vlanes, cudaStream_t s);

// NV12 hand-off (mc_preprocess.cu).  A 4:2:0 frame set: `lanes` frames, lane k's luma plane at y + k * lane_stride (h rows of
// w bytes, `pitch` apart) and its chroma at cb / cr + k * lane_stride, addressed as FrontArgs describes (h / 2 rows): NV12
// (interleaved Cb,Cr) or I420.  BGR frames are packed u8 BGR, lane k at bgr + k * bgr_step * h.  w and h are even.
struct Nv12Planes {
    const uint8_t* y = nullptr;
    const uint8_t* cb = nullptr;
    const uint8_t* cr = nullptr;
    size_t pitch = 0, cpitch = 0, lane_stride = 0;
    int cstep = kNv12ChromaStep;
};
// cvtColor(YUV2BGR_NV12) (I420: YUV2BGR_I420, the same arithmetic) of every lane
cudaError_t launch_nv12_to_bgr(const Nv12Planes& in, int w, int h, int lanes, uint8_t* bgr, size_t bgr_step, cudaStream_t s);
// cvtColor(BGR2YUV_I420) of every lane whose flag is set (flags: one byte per lane, or null for all), chroma interleaved
cudaError_t launch_bgr_to_nv12(const uint8_t* bgr, size_t bgr_step, int w, int h, int lanes, const uint8_t* flags,
                               uint8_t* y, uint8_t* uv, size_t pitch, size_t lane_stride, cudaStream_t s);

// The export canvas (mc_preprocess.cu): Exporter.cpp's compose(original, cur, split) over virtual lanes, its labels as
// the handle's overlay (mc_set_overlay): per-pixel u8 tone maps inside at most kOverlayRects disjoint canvas rects.
// A pane source holds virtual lane v's frame at p + v * lane_stride (4:2:0: its chroma at cb / cr + v * lane_stride,
// addressed as FrontArgs describes; RGB: its B, G and R channel bases at p, cb and cr + v * lane_stride, pixel step cstep).
struct PaneSrc {
    const uint8_t* p = nullptr;
    const uint8_t* cb = nullptr;
    size_t step = 0, lane_stride = 0;
    int kind = FRONT_BGR;           // FrontSrc: BGR, gray (expanded as GRAY2BGR), 4:2:0 or YUYV / UYVY (converted as cvtColor);
                                    // RGB for the front only (the compose kernel reads an RGB source's BGR tap)
    const uint8_t* cr = nullptr;
    size_t cpitch = 0;
    int cstep = kNv12ChromaStep;
};
// Which frame is virtual lane v's `cur` pane
enum ComposeOp : uint8_t { COMPOSE_SKIP = 0, COMPOSE_MAGNIFIED = 1, COMPOSE_FALLBACK = 2 };
constexpr int kOverlayRects = 2;    // MC_OVERLAY_MAX_RECTS
struct OverlayRect {
    int x = 0, y = 0, w = 0, h = 0;   // on the canvas
    const uint16_t* index = nullptr;  // device: h rows of w map indices
};
struct ComposeArgs {
    PaneSrc src[3];                 // the original pane, the magnifier's output, the fallback `cur` (front output or input)
    const uint8_t* ops = nullptr;   // ComposeOp per virtual lane; null: every lane MAGNIFIED
    int split = 0;                  // mc_split: the original pane is read only when it is not MC_SPLIT_NONE
    int w = 0, h = 0;               // pane size: even and > 0
    int format = 0;                 // mc_canvas_format; NV12 and I420 are told apart by cr
    uint8_t* data = nullptr;        // BGR / RGB canvas, luma plane or R plane of virtual lane 0
    uint8_t* uv = nullptr;          // NV12: Cb,Cr plane of virtual lane 0; I420: its Cb plane; RGB_PLANAR: its G plane
    uint8_t* cr = nullptr;          // I420: Cr plane of virtual lane 0, rows pitch / 2 apart in both chroma planes;
                                    // RGB_PLANAR: its B plane; NV12: null
    size_t pitch = 0, lane_stride = 0;
    int ov_rects = 0;               // the overlay: 0 .. kOverlayRects rects; 0 leaves every canvas as composed
    OverlayRect ov[kOverlayRects];
    const uint8_t* ov_map = nullptr;   // device: the tone maps, 256 bytes each
    int vec_src = 0, vec_out = 0, pane_blocks = 0;   // set by launch_compose
};
cudaError_t launch_compose(ComposeArgs a, int vlanes, cudaStream_t s);

// plane copy helpers
cudaError_t launch_copy_planes(float* dst, const float* src, size_t n, cudaStream_t s);

}  // namespace mc
