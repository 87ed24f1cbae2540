// The handle behind the C ABI: an H100-resident twin of livim::MagnificationProcessor
// (reference src/processing/MagnificationProcessor.cpp:10-67) — level clamp, structural reset,
// mode dispatch, passthrough decisions — plus device memory, streams and the pinned pipeline.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <deque>
#include <initializer_list>
#include <new>
#include <optional>
#include <string>
#include <vector>

#include "../../include/magcore_b200.h"
#include "mc_internal.h"
#include "mc_modes.h"

using namespace mc;

namespace {
thread_local std::string g_create_error;

// A grow-only device buffer of T, freed with its owner.  grow(need) frees the old allocation before it allocates the
// larger one.
template <class T = uint8_t>
struct DeviceBuffer {
    T* p = nullptr;
    size_t n = 0;   // capacity in T
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    ~DeviceBuffer() { if (p) cudaFree(p); }
    cudaError_t grow(size_t need) {
        if (need <= n) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        const cudaError_t e = cudaMalloc((void**)&p, need * sizeof(T));
        if (e == cudaSuccess) n = need;
        return e;
    }
};

// A grow-only pinned host buffer, freed with its owner.  grow(need) frees the old allocation before it allocates the
// larger one.
struct PinnedBuffer {
    uint8_t* p = nullptr;
    size_t n = 0;
    PinnedBuffer() = default;
    PinnedBuffer(const PinnedBuffer&) = delete;
    PinnedBuffer& operator=(const PinnedBuffer&) = delete;
    ~PinnedBuffer() { if (p) cudaFreeHost(p); }
    cudaError_t grow(size_t need) {
        if (need <= n) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; n = 0;
        const cudaError_t e = cudaHostAlloc((void**)&p, need, cudaHostAllocDefault);
        if (e == cudaSuccess) n = need;
        return e;
    }
};

// A frame set: one plane per lane (BGR or gray: height rows of w * c bytes), two (NV12: height luma rows and height / 2
// Cb,Cr rows of w bytes) or three (I420: height luma rows of w bytes, height / 2 rows of w / 2 bytes in each chroma plane).
// Plane k's rows hold row[k] bytes and are pitch[k] apart; lane l starts l * lane_stride after lane 0, in every plane.
struct Planes {
    static constexpr int kMax = 3;
    uint8_t* base[kMax] = {};
    size_t rows[kMax] = {};   // rows per lane; 0: no such plane
    size_t row[kMax] = {}, pitch[kMax] = {};
    size_t lane_stride = 0;

    size_t lane_rows() const { return rows[0] + rows[1] + rows[2]; }
    size_t lane_bytes() const { return rows[0] * row[0] + rows[1] * row[1] + rows[2] * row[2]; }
    // the same shape packed at `p`: no row padding, each plane right after the one before, lanes back to back
    Planes packed(uint8_t* p) const {
        Planes q;
        for (int k = 0; k < kMax && rows[k]; ++k) {
            q.base[k] = p; q.rows[k] = rows[k]; q.row[k] = q.pitch[k] = row[k];
            p += rows[k] * row[k];
        }
        q.lane_stride = lane_bytes();
        return q;
    }
    // `lanes` consecutive lanes are one run of lanes * lane_rows() rows of row[0] bytes, pitch[0] apart
    bool one_run(size_t lanes) const {
        size_t at = 0;
        for (int k = 0; k < kMax && rows[k]; ++k) {
            if (row[k] != row[0] || pitch[k] != pitch[0] || base[k] != base[0] + at) return false;
            at += rows[k] * pitch[0];
        }
        return lanes == 1 || lane_stride == at;
    }
    // the bytes of `lanes` consecutive lanes lie back to back without a gap: one linear copy moves them
    bool dense(size_t lanes) const {
        size_t at = 0;
        for (int k = 0; k < kMax && rows[k]; ++k) {
            if (pitch[k] != row[k] || base[k] != base[0] + at) return false;
            at += rows[k] * row[k];
        }
        return lanes == 1 || lane_stride == at;
    }
};

Planes bgr_planes(const uint8_t* p, int w, int hh, int c, size_t step) {
    return Planes{{const_cast<uint8_t*>(p)}, {(size_t)hh}, {(size_t)w * c}, {step}, step * hh};
}
Planes nv12_planes(const mc_nv12& f, int w, int hh) {
    return Planes{{f.y, f.uv}, {(size_t)hh, (size_t)hh / 2}, {(size_t)w, (size_t)w}, {f.pitch, f.pitch}, f.lane_stride};
}
mc_nv12 nv12_of(const Planes& f) { return mc_nv12{f.base[0], f.base[1], f.pitch[0], f.lane_stride}; }
// the luma plane and chroma addressing (mc_internal.h) of 4:2:0 planes: NV12 with two planes, I420 with three
Nv12Planes yuv420_of(const Planes& f) {
    if (!f.rows[2]) return Nv12Planes{f.base[0], f.base[1], f.base[1] + 1, f.pitch[0], f.pitch[0], f.lane_stride, kNv12ChromaStep};
    return Nv12Planes{f.base[0], f.base[1], f.base[2], f.pitch[0], f.pitch[1], f.lane_stride, kI420ChromaStep};
}

// The source frames of a call: u8 BGR or gray, 4:2:0 planes (NV12, or I420 with three planes), packed 4:2:2 frames or
// RGB frames (packed in one plane, planar in three), virtual lane v at v * planes.lane_stride.  Only these helpers tell
// the formats apart.
struct Source {
    static constexpr int kBadOrder = FRONT_RGB + 1;    // a 4:2:2 frame of an order out of range: refused by check()
    int kind = FRONT_BGR;                               // FrontSrc, the front's `src`
    int w = 0, hh = 0, channels = 3;                    // 4:2:0 and 4:2:2 frames stand for BGR ones
    Planes planes;
    const char* missing = nullptr;   // the call's mc_nv12 / mc_yuv420p / mc_yuv422 / mc_rgb is NULL: its error comes first
    bool i420 = false;               // 4:2:0 in three planes (mc_yuv420p)
    int layout = MC_RGB_RGB;         // FRONT_RGB: the mc_rgb_layout

    // bytes per pixel of an RGB layout's plane: 3 or 4 packed, 1 planar (an out-of-range layout is refused by check())
    static int rgb_pstep(int layout) { return layout == MC_RGB_RGB ? 3 : layout == MC_RGB_PLANAR ? 1 : 4; }

    static Source bgr(const uint8_t* in, int w, int hh, int c, size_t step) {
        return Source{c == 3 ? FRONT_BGR : FRONT_GRAY, w, hh, c, bgr_planes(in, w, hh, c, step)};
    }
    static Source nv12(const mc_nv12* f, int w, int hh) {
        return f ? Source{FRONT_NV12, w, hh, 3, nv12_planes(*f, w, hh)} : Source{FRONT_NV12, w, hh, 3, {}, "NV12 plane is null"};
    }
    static Source yuv420p(const mc_yuv420p* f, int w, int hh) {
        if (!f) return Source{FRONT_NV12, w, hh, 3, {}, "I420 frame is null", true};
        const size_t ch = (size_t)std::max(hh, 0) / 2, cw = (size_t)std::max(w, 0) / 2;
        return Source{FRONT_NV12, w, hh, 3,
                      Planes{{f->y, f->u, f->v}, {(size_t)std::max(hh, 0), ch, ch}, {(size_t)std::max(w, 0), cw, cw},
                             {f->pitch, f->chroma_pitch, f->chroma_pitch}, f->lane_stride},
                      nullptr, true};
    }
    static Source rgb(const mc_rgb* f, int w, int hh) {
        if (!f) return Source{FRONT_RGB, w, hh, 3, {}, "RGB frame is null"};
        const size_t rows = (size_t)std::max(hh, 0), row = (size_t)std::max(w, 0) * rgb_pstep(f->layout);
        Source s{FRONT_RGB, w, hh, 3};
        s.layout = f->layout;
        if (f->layout == MC_RGB_PLANAR)
            s.planes = Planes{{f->data, f->g, f->b}, {rows, rows, rows}, {row, row, row}, {f->pitch, f->pitch, f->pitch}, f->lane_stride};
        else
            s.planes = Planes{{f->data}, {rows}, {row}, {f->pitch}, f->lane_stride};
        return s;
    }
    static Source yuv422(const mc_yuv422* f, int w, int hh) {
        if (!f) return Source{FRONT_YUYV, w, hh, 3, {}, "YUYV frame is null"};
        const int kind = f->order == MC_YUV422_YUYV || f->order == MC_YUV422_UYVY ? FRONT_YUYV + f->order : kBadOrder;
        return Source{kind, w, hh, 3, Planes{{f->data}, {(size_t)hh}, {(size_t)2 * w}, {f->pitch}, f->lane_stride}};
    }

    // BGR or gray frames, which the magnifier reads where they are
    bool bgr_or_gray() const { return kind == FRONT_BGR || kind == FRONT_GRAY; }
    // the identity: no BGR or gray frame (NV12 and 4:2:2 frames are checked instead)
    bool empty() const { return bgr_or_gray() && (!planes.base[0] || w <= 0 || hh <= 0); }
    // the 4:2:2 and RGB conversions are a front stage that always runs: the front writes its BGR frame where a BGR source
    // would leave the result to the input
    bool converts() const { return kind >= FRONT_YUYV; }
    // the compose kernel reads the original pane from the front's BGR tap rather than from the frames: RGB, whose channel
    // swap does not fit the kernel's registers (the tap is the frame the front writes for the magnifier anyway)
    bool composes_from_tap() const { return kind == FRONT_RGB; }
    // the source's argument errors for `vl` virtual lanes -> an error text, or null
    const char* check(size_t vl) const {
        if (i420) {
            if (w < 2 || hh < 2 || (w & 1) || (hh & 1)) return "I420 width and height must be even and >= 2";
            if (!planes.base[0] || !planes.base[1] || !planes.base[2]) return "I420 plane is null";
            if (planes.pitch[0] < (size_t)w) return "I420 pitch < width";
            if (planes.pitch[1] < (size_t)w / 2) return "I420 chroma_pitch < width / 2";
            if (vl > 1 && planes.lane_stride < planes.pitch[0] * hh) return "I420 lane_stride < pitch * height";
            return nullptr;
        }
        if (kind == FRONT_NV12) {
            if (w < 2 || hh < 2 || (w & 1) || (hh & 1)) return "NV12 width and height must be even and >= 2";
            if (!planes.base[0] || !planes.base[1]) return "NV12 plane is null";
            if (planes.pitch[0] < (size_t)w) return "NV12 pitch < width";
            if (vl > 1 && planes.lane_stride < planes.pitch[0] * hh) return "NV12 lane_stride < pitch * height";
            return nullptr;
        }
        if (kind == FRONT_RGB) {
            if (!planes.base[0]) return "RGB data is null";
            if (layout < MC_RGB_RGB || layout > MC_RGB_PLANAR) return "RGB layout out of range";
            if (layout == MC_RGB_PLANAR && (!planes.base[1] || !planes.base[2])) return "RGB plane is null";
            if (w < 1 || hh < 1) return "RGB width and height must be >= 1";
            if (planes.pitch[0] < planes.row[0]) return "RGB pitch < width * bytes per pixel";
            if (vl > 1 && planes.lane_stride < planes.pitch[0] * hh) return "RGB lane_stride < pitch * height";
            return nullptr;
        }
        if (converts()) {
            if (!planes.base[0]) return "YUYV frame is null";
            if (kind == kBadOrder) return "YUYV order out of range";
            if (w < 2 || (w & 1) || hh < 1) return "YUYV width must be even and >= 2, height >= 1";
            if (planes.pitch[0] < (size_t)2 * w) return "YUYV pitch < 2 * width";
            if (vl > 1 && planes.lane_stride < planes.pitch[0] * hh) return "YUYV lane_stride < pitch * height";
            return nullptr;
        }
        return !empty() && planes.pitch[0] < planes.row[0] ? "step too small" : nullptr;
    }
    // the frames as the front and the compose kernel read them
    PaneSrc pane() const {
        if (kind == FRONT_RGB) {   // the B, G and R channel bases (mc_internal.h)
            uint8_t* const* b = planes.base;
            const size_t pitch = planes.pitch[0];
            if (layout == MC_RGB_PLANAR) return PaneSrc{b[2], b[1], pitch, planes.lane_stride, kind, b[0], pitch, 1};
            const bool bgra = layout == MC_RGB_BGRA;
            return PaneSrc{b[0] + (bgra ? 0 : 2), b[0] + 1, pitch, planes.lane_stride, kind, b[0] + (bgra ? 2 : 0), pitch,
                           rgb_pstep(layout)};
        }
        if (kind != FRONT_NV12) return PaneSrc{planes.base[0], nullptr, planes.pitch[0], planes.lane_stride, kind};
        const Nv12Planes f = yuv420_of(planes);
        return PaneSrc{f.y, f.cb, f.pitch, f.lane_stride, kind, f.cr, f.cpitch, f.cstep};
    }
    // the same frames at `p` (a pipeline slot's packed device copy)
    Source on(const Planes& p) const { Source s = *this; s.planes = p; return s; }
};

// A slot's output frame sets: the processed frames and, for chain submits, the original tap.  Set k sits at
// out_ofs(k) in the slot's device output and in its pinned output staging.
constexpr int kOutSets = 2;

// One in-flight frame set of the pinned pipeline: one frame of every lane, or a clip of `frames` frames of every lane
// (virtual lane v = t * lanes + k).  The per-lane arrays hold frames * lanes entries.  Frees what it holds.
struct Slot {
    PinnedBuffer h_in, h_out;                    // pinned staging (packed), grown only for pageable inputs / outputs
    DeviceBuffer<> d_in, d_out;                  // device frames (packed)
    cudaEvent_t ev_in = nullptr, ev_k = nullptr, ev_done = nullptr;
    int produced = 0;
    std::vector<uint8_t> lane_produced;          // per virtual lane: the magnifier produced
    uint8_t* flags_out = nullptr;                // the caller's copy of lane_produced, written by mc_collect (null: none)
    Planes out[kOutSets];                        // the caller's destinations (base null: none)
    size_t out_ofs[kOutSets] = {};
    std::vector<uint8_t> written[kOutSets];      // per set and virtual lane: its bytes of out[k] are written
    bool direct_out[kOutSets] = {};              // D2H goes straight into out[k] (pinned)
    ~Slot() {
        for (cudaEvent_t e : {ev_in, ev_k, ev_done}) if (e) cudaEventDestroy(e);
    }
};

// A normalised ROI {x, y, w, h}: pre_roiX / Y / W / H of mc_params
using Roi = std::array<float, 4>;
constexpr Roi kFullRoi = {0.f, 0.f, 1.f, 1.f};
Roi roi_of(const mc_params& p) { return {p.pre_roiX, p.pre_roiY, p.pre_roiW, p.pre_roiH}; }
// exact != on every field, as the reference's fingerprint compares (IProcessor.hpp:35-39): a NaN never equals
bool roi_differs(const Roi& a, const Roi& b) { return a[0] != b[0] || a[1] != b[1] || a[2] != b[2] || a[3] != b[3]; }
}  // namespace

struct mc_handle {
    int device = 0;
    int lanes = 1;
    cudaStream_t stream = nullptr, s_in = nullptr, s_out = nullptr;
    DeviceTables tables;
    std::string err;
    uint64_t launches = 0;

    // StructuralTracker (MagnifyCore.hpp:45-80): the handle's part of the fingerprint, and per lane the ROI of its
    // effective params (mc_set_lane_roi), so that a lane whose ROI alone moves restarts alone
    int t_mode = MC_MODE_NONE, t_levels = -1, t_channels = -1, t_w = 0, t_h = 0;
    int t_down = 1, t_roi = 0;
    std::vector<Roi> t_lroi;
    std::vector<uint8_t> roi_moved;   // per frame call: lanes whose ROI fingerprint changes (tracker_plan)

    Options opt;
    Profiler prof;
    int depth = 3;

    MotionMode motion;
    ColorMode color;
    RieszMode riesz;

    DeviceBuffer<float> float_out;   // keep_float_output: the tap of the last frame call

    // chain calls: the front's staging (preprocessed frames when no tap is wanted, gray frames), the held-lane flags, and
    // the INTER_AREA tap tables with the geometry (rw, dw, rh, dh) they were built for and their host copy
    DeviceBuffer<> f_pre, f_gray, f_flags, f_tabs;
    int f_tab_key[4] = {-1, -1, -1, -1};
    size_t f_tab_ofs[3] = {0, 0, 0};   // byte offsets of the y taps, x offsets, y offsets
    std::vector<uint8_t> f_tabs_host, f_flags_host;
    // chain compose calls: the magnifier's output and the ComposeOp of every virtual lane, with its host copy
    DeviceBuffer<> x_mag, x_ops;
    std::vector<uint8_t> x_ops_host;
    // the export canvas's overlay (mc_set_overlay): configuration, kept across resets.  ov_dev holds the maps, then each
    // rect's index plane at byte offset ofs[i]
    struct Overlay {
        bool set = false;
        int cw = 0, ch = 0, rects = 0;
        OverlayRect rect[kOverlayRects];
        size_t ofs[kOverlayRects] = {};
    } ov;
    DeviceBuffer<> ov_dev;
    std::vector<uint8_t> ov_host;

    // mc_process_clip device staging: the clip's frames in and out
    DeviceBuffer<> k_in, k_out;

    // NV12 calls: the magnifier's BGR input and output, and the produced flags of a call where only some lanes produced
    DeviceBuffer<> n_in, n_out, n_flags;

    // pipeline
    std::vector<Slot> slots;
    std::deque<int> inflight;
    int next_slot = 0;

    // Lane lifecycle: per lane, whether it has temporal state (cleared by mc_reset, structural changes, mode None and the
    // error path, or for one lane by mc_restart_lane) and whether it is held (mc_hold_lane; sticky).  A frame call turns
    // them into one LaneOp per lane.
    std::vector<uint8_t> has_state, hold, ops;
    std::vector<uint8_t> lane_produced;   // of the frame most recently returned / collected
    uint8_t* d_ops = nullptr;             // device copy of a mixed frame's ops (the mode uploads it on the handle's stream)
    // Per-lane parameters (mc_set_lane_params): configuration, kept across resets.  lane_eff holds each lane's effective
    // parameters of the current frame call.
    std::vector<mc_lane_params> lane_lp;
    std::vector<uint8_t> lane_lp_set;
    int n_lane_lp = 0;
    std::vector<mc_params> lane_eff;
    std::vector<uint8_t> lane_lost;   // per frame call: lanes whose state the mode dropped
    // Per-lane ROIs (mc_set_lane_roi): configuration, kept across resets
    std::vector<Roi> lane_roi;
    std::vector<uint8_t> lane_roi_set;
    int n_lane_roi = 0;
    // chain calls whose lanes crop at different origins: one origin per virtual lane, and its host copy
    DeviceBuffer<int2> f_org;
    std::vector<int2> f_org_host;
    // mc_save_lane / mc_load_lane: pinned staging of a blob's planes when the caller's buffer is pageable (grow-only)
    PinnedBuffer lane_stage;
};

namespace {
// ---- exception firewall of the C ABI ------------------------------------------------------------------------
// include/magcore_b200.h promises that no C++ exception crosses the boundary (the reference's own firewall,
// ProcessingChain.cpp:50-62, sits ABOVE the adapter and only understands what the adapter rethrows).  Every
// extern "C" entry with a body that can allocate is a function-try-block ending in on_exception().
thread_local int g_inject_throw = 0;   // test hook (mc_debug_inject_exception): >0 = throw at the n-th guarded entry

inline void debug_maybe_throw() {
    if (g_inject_throw > 0 && --g_inject_throw == 0) throw std::bad_alloc();
}

void reset_modes(mc_handle* h);
void tracker_reset(mc_handle* h);

mc_status on_exception(mc_handle* h) noexcept {
    const char* what = "unknown C++ exception";
    std::string buf;
    try { throw; }
    catch (const std::bad_alloc&) { what = "out of host memory (std::bad_alloc)"; }
    catch (const std::exception& e) {
        try { buf = std::string("C++ exception: ") + e.what(); what = buf.c_str(); } catch (...) {}
    }
    catch (...) {}
    try {
        if (h) {
            h->err = what;
            // the recovery contract of ProcessingChain.cpp:50-62: temporal state may be half-updated, drop it
            reset_modes(h);
            tracker_reset(h);
        } else {
            g_create_error = what;
        }
    } catch (...) {}
    return MC_ERR_INTERNAL;
}
}  // namespace

#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            h->err = std::string(#call) + ": " + cudaGetErrorString(e__);                         \
            return MC_ERR_CUDA;                                                                   \
        }                                                                                         \
    } while (0)

namespace {

void tracker_disable(mc_handle* h) {
    h->t_mode = MC_MODE_NONE; h->t_levels = -1; h->t_channels = -1; h->t_w = 0; h->t_h = 0;
}
void tracker_reset(mc_handle* h) {
    tracker_disable(h);
    h->t_down = 1; h->t_roi = 0;
    h->t_lroi.assign((size_t)h->lanes, kFullRoi);
}
// The handle's part of the fingerprint: everything but the ROI rectangle, which each lane keeps (t_lroi).
bool tracker_changes(const mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    return p->mode != h->t_mode || lv != h->t_levels || w != h->t_w || hh != h->t_h ||
           ch != h->t_channels || p->pre_downscale != h->t_down || (p->pre_roiEnabled != 0) != (h->t_roi != 0);
}
void tracker_set(mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    h->t_mode = p->mode; h->t_levels = lv; h->t_w = w; h->t_h = hh; h->t_channels = ch;
    h->t_down = p->pre_downscale; h->t_roi = p->pre_roiEnabled != 0;
}
// Lane l's effective ROI: its override (mc_set_lane_roi), or the call's.
Roi lane_roi(const mc_handle* h, const mc_params& p, size_t l) { return h->lane_roi_set[l] ? h->lane_roi[l] : roi_of(p); }
// The fingerprint's verdict on a call: true when the handle resets structurally, because its own part changed or every
// lane's ROI did (a change of the call's ROI without overrides, as before lanes had their own).  Otherwise h->roi_moved
// flags the lanes whose ROI alone changed: each restarts alone, as its 1-lane twin would.  A held lane keeps its state and
// its fingerprint, because its twin skips the call: it is compared when the lane runs again, so a ROI moved and moved back
// during a hold restarts nothing.
bool tracker_plan(mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    const size_t lanes = (size_t)h->lanes;
    h->roi_moved.assign(lanes, 0);
    if (tracker_changes(h, p, lv, ch, w, hh)) return true;
    size_t n = 0;
    for (size_t l = 0; l < lanes; ++l) n += h->roi_moved[l] = roi_differs(lane_roi(h, *p, l), h->t_lroi[l]);
    if (n == lanes) return true;
    for (size_t l = 0; l < lanes; ++l) h->roi_moved[l] = h->roi_moved[l] && !h->hold[l];
    return false;
}
// tracker_plan, applied: true for a structural reset (the caller drops every lane's state); a running lane whose ROI alone
// moved loses its state here, and a Phase lane's next frame re-designs its filters at its framerate, as its twin's
// structural reset does.
bool tracker_update(mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    const bool change = tracker_plan(h, p, lv, ch, w, hh);
    if (change) tracker_set(h, p, lv, ch, w, hh);
    for (size_t l = 0; l < (size_t)h->lanes; ++l) {
        if (!change && !h->roi_moved[l]) continue;
        h->t_lroi[l] = lane_roi(h, *p, l);
        if (change) continue;
        h->has_state[l] = 0;
        h->riesz.redesign((int)l);
    }
    return change;
}

void reset_modes(mc_handle* h) {
    std::fill(h->has_state.begin(), h->has_state.end(), (uint8_t)0);
    h->motion.reset();
    h->color.reset();
    h->riesz.reset();
}

void free_slots(mc_handle* h) {
    h->slots.clear();
    h->inflight.clear();
    h->next_slot = 0;
}

// Slots with device buffers for `in_bytes` of input and `out_bytes` of output per frame set.  They are reallocated, never
// below their current sizes, only while nothing is in flight.  Their pinned staging is grown by submit_impl when a
// submit's buffers are pageable.
mc_status ensure_slots(mc_handle* h, size_t in_bytes, size_t out_bytes) {
    const bool have = (int)h->slots.size() == h->depth;
    if (have && h->slots[0].d_in.n >= in_bytes && h->slots[0].d_out.n >= out_bytes) return MC_OK;
    if (!h->inflight.empty()) {
        h->err = "pipeline geometry changed with frames in flight";
        return MC_ERR_INVALID;
    }
    if (have) {
        in_bytes = std::max(in_bytes, h->slots[0].d_in.n);
        out_bytes = std::max(out_bytes, h->slots[0].d_out.n);
    }
    free_slots(h);
    h->slots = std::vector<Slot>((size_t)h->depth);
    for (auto& s : h->slots) {
        CK(s.d_in.grow(in_bytes));
        CK(s.d_out.grow(out_bytes));
        CK(cudaEventCreateWithFlags(&s.ev_in, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&s.ev_k, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
    }
    return MC_OK;
}

bool is_pinned(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeHost;
}
bool is_pinned(const Planes& f) {
    for (int k = 0; k < Planes::kMax && f.rows[k]; ++k)
        if (!is_pinned(f.base[k])) return false;
    return true;
}

// Lane l of every plane, host to host, row by row.
void host_copy(const Planes& dst, const Planes& src, size_t l) {
    for (int k = 0; k < Planes::kMax; ++k)
        for (size_t r = 0; r < src.rows[k]; ++r)
            std::memcpy(dst.base[k] + l * dst.lane_stride + r * dst.pitch[k], src.base[k] + l * src.lane_stride + r * src.pitch[k],
                        src.row[k]);
}

// Lanes [a, b) of every plane between host and device: one plain copy when neither side has a gap between their bytes,
// one 2D copy when both sides hold them as one run of rows of one width, otherwise one 2D copy per plane and lane.
mc_status copy_planes(mc_handle* h, const Planes& dst, const Planes& src, size_t a, size_t b, cudaMemcpyKind kind, cudaStream_t s) {
    uint8_t* d = dst.base[0] + a * dst.lane_stride;
    const uint8_t* from = src.base[0] + a * src.lane_stride;
    if (dst.dense(b - a) && src.dense(b - a)) {
        CK(cudaMemcpyAsync(d, from, (b - a) * src.lane_bytes(), kind, s));
        return MC_OK;
    }
    if (dst.one_run(b - a) && src.one_run(b - a)) {
        CK(cudaMemcpy2DAsync(d, dst.pitch[0], from, src.pitch[0], src.row[0], (b - a) * src.lane_rows(), kind, s));
        return MC_OK;
    }
    for (size_t l = a; l < b; ++l)
        for (int k = 0; k < Planes::kMax; ++k)
            if (src.rows[k])
                CK(cudaMemcpy2DAsync(dst.base[k] + l * dst.lane_stride, dst.pitch[k], src.base[k] + l * src.lane_stride, src.pitch[k],
                                     src.row[k], src.rows[k], kind, s));
    return MC_OK;
}

// Without option "color_lane_lifecycle" a multi-lane Color handle keeps its lanes in lock-step: a frame call while a lane
// is held, or restarted while others run (mc_restart_lane, or its own ROI moved), is MC_ERR_UNSUPPORTED, checked before
// any state changes.
mc_status color_lane_check(mc_handle* h, const mc_params* p, int levels, int channels, int w, int hh) {
    if (h->opt.color_lane_lifecycle) return MC_OK;
    const bool change = tracker_plan(h, p, levels, channels, w, hh);
    int n_hold = 0, n_state = 0;
    for (size_t l = 0; l < (size_t)h->lanes; ++l) {
        n_hold += h->hold[l] != 0;
        n_state += h->has_state[l] && !h->roi_moved[l];
    }
    if (n_hold) { h->err = "Color mode cannot hold a lane of a multi-lane handle"; return MC_ERR_UNSUPPORTED; }
    if (!change && n_state != 0 && n_state != h->lanes) {
        h->err = "Color mode cannot restart one lane of a multi-lane handle while the others run";
        return MC_ERR_UNSUPPORTED;
    }
    return MC_OK;
}

// Each lane's effective parameters: the call's, with the six fields of the lane's override (mc_set_lane_params).  *q gets
// lane 0's; returns the `lanes` of them when they differ and null when every lane's are *q.  "Differ" is bitwise: +0 and
// -0 (or two NaNs) can step the temporal state into different bits, so only identical fields share the scalar path.
bool same_lane_fields(const mc_params& a, const mc_params& b) {
    static_assert(offsetof(mc_params, framerate) - offsetof(mc_params, amplification) == 5 * sizeof(double), "six adjacent doubles");
    return std::memcmp(&a.amplification, &b.amplification, 6 * sizeof(double)) == 0;
}
const mc_params* effective_params(mc_handle* h, const mc_params& p, mc_params* q) {
    *q = p;
    if (h->n_lane_lp == 0) return nullptr;
    h->lane_eff.assign((size_t)h->lanes, p);
    bool same = true;
    for (size_t l = 0; l < (size_t)h->lanes; ++l) {
        mc_params& e = h->lane_eff[l];
        if (h->lane_lp_set[l]) {
            const mc_lane_params& o = h->lane_lp[l];
            e.amplification = o.amplification; e.coWavelength = o.coWavelength; e.coLow = o.coLow; e.coHigh = o.coHigh;
            e.chromAttenuation = o.chromAttenuation; e.framerate = o.framerate;
        }
        same = same && same_lane_fields(e, h->lane_eff[0]);
    }
    *q = h->lane_eff[0];
    return same ? nullptr : h->lane_eff.data();
}

// Color lanes whose effective parameters differ need option color_lane_lifecycle: MC_ERR_UNSUPPORTED otherwise.
mc_status lane_params_check(mc_handle* h, const mc_params& p) {
    mc_params q;
    if (p.mode == MC_MODE_COLOR && !h->opt.color_lane_lifecycle && effective_params(h, p, &q)) {
        h->err = "Color lanes with different parameters (mc_set_lane_params) need option color_lane_lifecycle";
        return MC_ERR_UNSUPPORTED;
    }
    return MC_OK;
}

// The body of MagnificationProcessor::process on device-resident frames.
// lane_produced: `lanes` per-lane flags (written).  frames > 1: a clip of that many consecutive
// frames of every lane, [t][lane] in the lane stride, with frames * lanes flags.
mc_status process_device_impl(mc_handle* h, const uint8_t* d_in, int w, int hh, int channels, size_t in_step,
                              const mc_params* p, uint8_t* d_out, size_t out_step, int* produced, uint8_t* lane_produced,
                              int frames = 1) {
    const size_t n_flags = (size_t)frames * h->lanes;
    *produced = 0;
    std::fill(lane_produced, lane_produced + n_flags, (uint8_t)0);
    debug_maybe_throw();
    if (!p) { h->err = "params is null"; return MC_ERR_INVALID; }
    // Identity when disabled / empty; free state so a later re-enable starts cleanly (:21-29).
    if (p->mode == MC_MODE_NONE || d_in == nullptr || w <= 0 || hh <= 0) {
        if (h->t_mode != MC_MODE_NONE) {
            reset_modes(h);
            tracker_disable(h);
        }
        return MC_OK;
    }
    if (p->mode < 0 || p->mode > MC_MODE_NONE) { h->err = "bad mode"; return MC_ERR_INVALID; }
    if (channels != 1 && channels != 3) { h->err = "channels must be 1 or 3"; return MC_ERR_INVALID; }
    if (d_out == nullptr) { h->err = "output pointer is null"; return MC_ERR_INVALID; }
    if (in_step < (size_t)w * channels || out_step < (size_t)w * channels) { h->err = "step too small"; return MC_ERR_INVALID; }
    const int max_levels = calculate_max_levels(w, hh);  // :32-33
    if (max_levels < 1) return MC_OK;
    const int levels = std::min(std::max((int)p->levels, 1), max_levels);  // :34
    mc_status st = lane_params_check(h, *p);
    if (st != MC_OK) return st;
    mc_params q;
    const mc_params* lane_params = effective_params(h, *p, &q);
    p = &q;
    if (p->mode == MC_MODE_COLOR) {
        // A held 1-lane handle skips the call: its window stays as it is.
        if (h->lanes == 1 && h->hold[0]) return MC_OK;
        const mc_status st = color_lane_check(h, p, levels, channels, w, hh);
        if (st != MC_OK) return st;
    }
    if (tracker_update(h, p, levels, channels, w, hh)) reset_modes(h);      // :39-43
    int n_first = 0;
    for (int l = 0; l < h->lanes; ++l) {
        const uint8_t op = h->hold[(size_t)l] ? LANE_HOLD : h->has_state[(size_t)l] ? LANE_RUN : LANE_FIRST;
        h->ops[(size_t)l] = op;
        n_first += op == LANE_FIRST;
    }
    if (p->mode == MC_MODE_COLOR && n_first == h->lanes) h->color.reset();   // every lane restarted: a fresh window

    FrameIO io;
    io.in = d_in; io.in_step = in_step; io.in_lane_stride = in_step * (size_t)hh;
    io.out = d_out; io.out_step = out_step; io.out_lane_stride = out_step * (size_t)hh;
    io.w = w; io.h = hh; io.channels = channels; io.lanes = h->lanes;

    if (h->opt.keep_float_output) CK(h->float_out.grow((size_t)h->lanes * w * hh * channels));

    bool held_lost = false;
    h->lane_lost.assign((size_t)h->lanes, 0);
    Options opt = h->opt;
    if (opt.profile_kernels) opt.lane_groups = 1;   // one launch chain: the events time one kernel at a time
    const ModeCtx ctx{.stream = h->stream, .tables = &h->tables, .launches = &h->launches, .err = &h->err, .opt = opt,
                      .float_out = opt.keep_float_output ? h->float_out.p : nullptr,
                      .prof = opt.profile_kernels ? &h->prof : nullptr,
                      .lane_ops = h->ops.data(), .d_lane_ops = h->d_ops, .lane_produced = lane_produced, .held_lost = &held_lost,
                      .lane_params = lane_params, .lane_lost = h->lane_lost.data()};
    switch (p->mode) {
        case MC_MODE_LAPLACE: st = h->motion.process(ctx, io, *p, levels, produced, frames); break;
        case MC_MODE_COLOR: st = h->color.process(ctx, io, *p, levels, produced, frames); break;
        case MC_MODE_PHASE: st = h->riesz.process(ctx, io, *p, levels, produced, frames); break;
        default: break;
    }
    if (st != MC_OK) {
        // mirror the reference's recovery contract (ProcessingChain.cpp:50-62): state may be
        // half-updated, so drop it; the caller shows the input frame.
        reset_modes(h);
        tracker_reset(h);
        *produced = 0;
        std::fill(lane_produced, lane_produced + n_flags, (uint8_t)0);
        return st;
    }
    for (int l = 0; l < h->lanes; ++l) {
        if (h->ops[(size_t)l] != LANE_HOLD) h->has_state[(size_t)l] = 1;
        else if (held_lost || h->lane_lost[(size_t)l]) h->has_state[(size_t)l] = 0;
    }
    return st;
}

// One frame set into the pipeline: one frame of every lane, or with frames > 1 a clip of `frames` frames of every lane
// (virtual lane v = t * lanes + k at v * lane_stride of `in` and of each out[k]).  `in` is uploaded on the input stream
// into the next slot's packed device copy: directly when it is pinned, through the slot's pinned staging when not.
// `run(d_in, d_out, produced, lane_produced, written)` then fills the slot's packed output sets d_out[k] (the shapes of
// out[k], which may differ from `in`'s) on the handle's stream (with no buffers when `in` is empty: the identity), and
// says per set which virtual lanes it wrote.  Only those are downloaded on the output stream, one copy per run of
// consecutive ones, into out[k] when it is pinned and into the staging, which mc_collect copies out, when not; the other
// lanes' bytes of out[k] stay as they are.  The slot's d_in and d_out are not overwritten before its copies and kernels
// ran: the next upload into them follows mc_collect of this frame set, which waits on ev_done.  The slots' output holds
// at least out_reserve bytes.  flags_out (frames * lanes bytes, or null) gets lane_produced at mc_collect.
template <class Run>
mc_status submit_impl(mc_handle* h, const Planes& in, const Planes (&out)[kOutSets], Run run, size_t out_reserve = 0,
                      int frames = 1, uint8_t* flags_out = nullptr) {
    const size_t vl = (size_t)frames * h->lanes, bytes = in.lane_bytes() * vl;
    size_t ofs[kOutSets], out_bytes = 0;
    for (int k = 0; k < kOutSets; ++k) {
        if (out[k].base[0] && out[k].pitch[0] < out[k].row[0]) { h->err = "out_step too small"; return MC_ERR_INVALID; }
        ofs[k] = out_bytes;
        out_bytes += (out[k].lane_bytes() * vl + 255) / 256 * 256;   // each set 256-byte aligned
    }
    mc_status st = ensure_slots(h, std::max<size_t>(bytes, 1), std::max<size_t>({out_bytes, out_reserve, 1}));
    if (st != MC_OK) return st;
    const int si = h->next_slot;
    Slot& s = h->slots[(size_t)si];
    // pinned staging only for what is pageable
    const bool pinned_in = bytes && is_pinned(in);
    if (bytes && !pinned_in) CK(s.h_in.grow(bytes));
    bool staged_out = false;
    for (int k = 0; k < kOutSets; ++k) {
        s.direct_out[k] = out[k].base[0] && is_pinned(out[k]);
        staged_out |= out[k].base[0] && !s.direct_out[k];
    }
    if (staged_out) CK(s.h_out.grow(out_bytes));
    s.produced = 0;
    s.lane_produced.assign(vl, 0);
    s.flags_out = flags_out;
    const Planes none;
    Planes d_out[kOutSets];
    for (int k = 0; k < kOutSets; ++k) {
        s.out[k] = out[k]; s.out_ofs[k] = ofs[k];
        s.written[k].assign(vl, 0);
        d_out[k] = out[k].lane_bytes() ? out[k].packed(s.d_out.p + ofs[k]) : none;
    }
    const Planes d_in = bytes ? in.packed(s.d_in.p) : none;
    if (bytes) {
        const Planes src = pinned_in ? in : in.packed(s.h_in.p);
        if (!pinned_in)
            for (size_t l = 0; l < vl; ++l) host_copy(src, in, l);
        if ((st = copy_planes(h, d_in, src, 0, vl, cudaMemcpyHostToDevice, h->s_in)) != MC_OK) return st;
        CK(cudaEventRecord(s.ev_in, h->s_in));
        CK(cudaStreamWaitEvent(h->stream, s.ev_in, 0));
    }
    int produced = 0;
    if ((st = run(d_in, d_out, &produced, s.lane_produced.data(), s.written)) != MC_OK) return st;
    s.produced = produced;
    bool download = false;
    for (int k = 0; k < kOutSets; ++k)
        download |= out[k].base[0] && std::any_of(s.written[k].begin(), s.written[k].end(), [](uint8_t x) { return x != 0; });
    if (download) {
        CK(cudaEventRecord(s.ev_k, h->stream));
        CK(cudaStreamWaitEvent(h->s_out, s.ev_k, 0));
        for (int k = 0; k < kOutSets; ++k) {
            if (!out[k].base[0]) continue;
            const Planes dst = s.direct_out[k] ? out[k] : out[k].packed(s.h_out.p + ofs[k]);
            st = for_each_run(vl, [&](size_t l) { return s.written[k][l] != 0; }, [&](size_t a, size_t b) {
                return copy_planes(h, dst, d_out[k], a, b, cudaMemcpyDeviceToHost, h->s_out);
            });
            if (st != MC_OK) return st;
        }
        CK(cudaEventRecord(s.ev_done, h->s_out));
    } else {
        CK(cudaEventRecord(s.ev_done, h->stream));
    }
    h->inflight.push_back(si);
    h->next_slot = (si + 1) % h->depth;
    return MC_OK;
}

// ---- lane state blobs (mc_save_lane / mc_load_lane) ----------------------------------------------------------------
constexpr char kBlobMagic[8] = {'M', 'C', 'L', 'A', 'N', 'E', 0, 0};
constexpr uint32_t kBlobVersion = 1;
// A blob's header.  The lane's state planes follow it, in the order the mode lists them (lane_planes), as dense rows.
struct LaneBlob {
    char magic[8];
    uint32_t version;
    uint32_t has_state;   // the lane's "has state" bit; a blob without state has no planes
    uint64_t bytes;       // the whole blob: header + planes
    // the structural key (tracker_changes) and, for Laplace, faithful_level0
    int32_t mode, levels, w, h, channels, pre_down, pre_roi, faithful;
    float roi[4];
    int32_t ab_bounded;   // Laplace: the handle's ab_bounded (L-only synthesis, DESIGN §4)
    int32_t count, head, mod;   // Color: the lane's window
    double design[15];    // Phase: the lane's RieszMode::Design (lo_freq, hi_freq, framerate, loA, loB, hiA, hiB)
};
static_assert(sizeof(LaneBlob) == 208, "no padding: every byte of a header is defined");
static_assert(sizeof(RieszMode::Design) == sizeof(LaneBlob::design), "Design is 15 doubles");

mc_params blob_key(const LaneBlob& b) {
    mc_params p{};
    p.mode = b.mode; p.pre_downscale = b.pre_down; p.pre_roiEnabled = b.pre_roi;
    p.pre_roiX = b.roi[0]; p.pre_roiY = b.roi[1]; p.pre_roiW = b.roi[2]; p.pre_roiH = b.roi[3];
    return p;
}

// Lane `lane`'s state planes for the blob's mode (Color: a window of the blob's length) -> their bytes
size_t lane_planes(mc_handle* h, const LaneBlob& b, int lane, std::vector<LanePlane>& out) {
    out.clear();
    if (b.has_state) {
        if (b.mode == MC_MODE_LAPLACE) h->motion.lane_planes(lane, out);
        else if (b.mode == MC_MODE_PHASE) h->riesz.lane_planes(lane, out);
        else if (b.mode == MC_MODE_COLOR) h->color.lane_planes(lane, b.mod, out);
    }
    size_t total = 0;
    for (const LanePlane& p : out) total += p.row_bytes * p.rows;
    return total;
}

// The planes between the device and `host` (the blob's plane bytes, dense) on the handle's stream, through the pinned
// staging when `host` is pageable; complete when it returns.
mc_status copy_lane_planes(mc_handle* h, const std::vector<LanePlane>& planes, size_t total, uint8_t* host, bool save) {
    const bool pinned = is_pinned(host);
    if (!pinned) CK(h->lane_stage.grow(total));
    uint8_t* base = pinned ? host : h->lane_stage.p;
    if (!pinned && !save) std::memcpy(base, host, total);
    size_t ofs = 0;
    for (const LanePlane& p : planes) {
        if (save) CK(cudaMemcpy2DAsync(base + ofs, p.row_bytes, p.ptr, p.pitch, p.row_bytes, p.rows, cudaMemcpyDeviceToHost, h->stream));
        else CK(cudaMemcpy2DAsync(p.ptr, p.pitch, base + ofs, p.row_bytes, p.row_bytes, p.rows, cudaMemcpyHostToDevice, h->stream));
        ofs += p.row_bytes * p.rows;
    }
    CK(cudaStreamSynchronize(h->stream));
    if (!pinned && save) std::memcpy(host, base, total);
    return MC_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int mc_abi_version(void) { return MC_ABI_VERSION; }

int mc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

void mc_params_default(mc_params* p) {
    if (!p) return;
    std::memset(p, 0, sizeof(*p));
    p->mode = MC_MODE_LAPLACE;
    p->levels = 4;
    p->framerate = 30.0;
    p->pre_downscale = 1;
    p->pre_roiW = 1.0f;
    p->pre_roiH = 1.0f;
}

static double hz_to_blend(double hz, double fps) {  // MagnificationParamsUi.hpp:29-34
    if (fps <= 0.0) fps = 30.0;
    if (hz <= 0.0) return 0.0;
    const double a = 1.0 - std::exp(-6.283185307179586 * hz / fps);
    return std::min(std::max(a, 0.0), 0.999999);
}

void mc_params_from_ui(mc_params* p, int mode, int amplification, double wavelength, double low_hz, double high_hz,
                       int chroma, int levels, double fps) {
    if (!p) return;
    mc_params_default(p);
    p->mode = mode;
    p->amplification = amplification;
    p->levels = levels;
    p->framerate = fps;
    switch (mode) {
        case MC_MODE_COLOR:
            p->coLow = low_hz; p->coHigh = high_hz;
            break;
        case MC_MODE_LAPLACE:
            p->coWavelength = wavelength * 10.0;
            p->coLow = hz_to_blend(low_hz, fps);
            p->coHigh = hz_to_blend(high_hz, fps);
            p->chromAttenuation = chroma / 100.0;
            break;
        case MC_MODE_PHASE:
            p->coWavelength = 100.0 - wavelength;
            p->coLow = low_hz; p->coHigh = high_hz;
            break;
        default: break;
    }
}

int mc_calculate_max_levels(int width, int height) { return calculate_max_levels(width, height); }
int mc_optimal_buffer_size(int fps) { return optimal_buffer_size(fps); }

mc_status mc_butterworth(unsigned order, double wn, double* a, double* b) try {
    debug_maybe_throw();
    if (!a || !b || order == 0 || order > 16) return MC_ERR_INVALID;
    std::vector<double> va, vb;
    butterworth(order, wn, va, vb);
    for (unsigned i = 0; i <= order; ++i) { a[i] = va[i]; b[i] = vb[i]; }
    return MC_OK;
} catch (...) { return on_exception(nullptr); }

mc_status mc_motion_gains(const mc_params* p, int levels, int width, int height, float* gains) try {
    debug_maybe_throw();
    if (!p || !gains || levels < 1) return MC_ERR_INVALID;
    std::vector<float> g;
    motion_gains(p->amplification, p->coWavelength, levels, width, height, g);
    for (int i = 0; i <= levels; ++i) gains[i] = g[(size_t)i];
    return MC_OK;
} catch (...) { return on_exception(nullptr); }

mc_status mc_create_lanes(int device, int lanes, mc_handle** out) try {
    // grid.z carries lanes * channels (<= 65535) and the Color min/max scratch is sized per lane
    if (!out || lanes < 1 || lanes > MC_MAX_LANES) { g_create_error = "bad arguments (1 <= lanes <= MC_MAX_LANES)"; return MC_ERR_INVALID; }
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device < 0 || device >= n) {
        cudaGetLastError();
        g_create_error = "no usable CUDA device (this core has no CPU fallback)";
        return MC_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9) {
        cudaGetLastError();
        g_create_error = "device is not sm_90-class; kernels are built for sm_90a only";
        return MC_ERR_NO_DEVICE;
    }
    debug_maybe_throw();
    mc_handle* h = new mc_handle();
    try {
    h->device = device;
    h->lanes = lanes;
    auto fail = [&](const char* what, cudaError_t e) {
        g_create_error = std::string(what) + ": " + cudaGetErrorString(e);
        mc_destroy(h);
        return MC_ERR_CUDA;
    };
    cudaError_t e;
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    if ((e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("stream", e);
    if ((e = cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking)) != cudaSuccess) return fail("stream", e);
    if ((e = cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking)) != cudaSuccess) return fail("stream", e);
    std::vector<LabLutCell> lut;
    build_lab_lut_cells(lut);
    std::vector<LabLutPack> pack;
    if (!lut.empty()) build_lab_lut_packs(lut, pack);
    if (pack.empty()) { g_create_error = "embedded Lab LUT missing"; mc_destroy(h); return MC_ERR_INVALID; }
    std::vector<float4> gam;
    build_inv_gamma_spline(gam);
    build_lab_inv_coeffs(h->tables.inv_coeffs);
    if ((e = cudaMalloc((void**)&h->tables.lab_lut, lut.size() * sizeof(LabLutCell))) != cudaSuccess) return fail("cudaMalloc lut", e);
    if ((e = cudaMalloc((void**)&h->tables.inv_gamma, gam.size() * sizeof(float4))) != cudaSuccess) return fail("cudaMalloc gamma", e);
    if ((e = cudaMemcpy(h->tables.lab_lut, lut.data(), lut.size() * sizeof(LabLutCell), cudaMemcpyHostToDevice)) != cudaSuccess) return fail("copy lut", e);
    if ((e = cudaMalloc((void**)&h->tables.lab_pack, pack.size() * sizeof(LabLutPack))) != cudaSuccess) return fail("cudaMalloc packed lut", e);
    if ((e = cudaMemcpy(h->tables.lab_pack, pack.data(), pack.size() * sizeof(LabLutPack), cudaMemcpyHostToDevice)) != cudaSuccess) return fail("copy packed lut", e);
    if ((e = cudaMemcpy(h->tables.inv_gamma, gam.data(), gam.size() * sizeof(float4), cudaMemcpyHostToDevice)) != cudaSuccess) return fail("copy gamma", e);
    h->motion.lanes = h->color.lanes = h->riesz.lanes = lanes;
    h->has_state.assign((size_t)lanes, 0);
    h->hold.assign((size_t)lanes, 0);
    h->ops.assign((size_t)lanes, 0);
    h->lane_produced.assign((size_t)lanes, 0);
    h->lane_lp.assign((size_t)lanes, mc_lane_params{});
    h->lane_lp_set.assign((size_t)lanes, 0);
    h->lane_roi.assign((size_t)lanes, kFullRoi);
    h->lane_roi_set.assign((size_t)lanes, 0);
    h->t_lroi.assign((size_t)lanes, kFullRoi);
    if ((e = cudaMalloc((void**)&h->d_ops, (size_t)lanes)) != cudaSuccess) return fail("cudaMalloc lane ops", e);
    *out = h;
    return MC_OK;
    } catch (...) { mc_destroy(h); throw; }
} catch (...) { return on_exception(nullptr); }

mc_status mc_create(int device, mc_handle** out) { return mc_create_lanes(device, 1, out); }

void mc_destroy(mc_handle* h) try {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->s_in) cudaStreamSynchronize(h->s_in);
    if (h->s_out) cudaStreamSynchronize(h->s_out);
    reset_modes(h);
    if (h->tables.lab_lut) cudaFree(h->tables.lab_lut);
    if (h->tables.lab_pack) cudaFree(h->tables.lab_pack);
    if (h->tables.inv_gamma) cudaFree(h->tables.inv_gamma);
    if (h->d_ops) cudaFree(h->d_ops);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->s_in) cudaStreamDestroy(h->s_in);
    if (h->s_out) cudaStreamDestroy(h->s_out);
    delete h;   // the pipeline slots and the scratch buffers free themselves
} catch (...) {}

/* test hook, not declared in the public header: the n-th guarded entry on this thread throws std::bad_alloc */
void mc_debug_inject_exception(int nth) { g_inject_throw = nth; }

mc_status mc_reset(mc_handle* h) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    reset_modes(h);
    tracker_reset(h);
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_restart_lane(mc_handle* h, int lane) try {
    if (!h) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    if (h->lanes == 1) return mc_reset(h);
    h->has_state[(size_t)lane] = 0;   // taken into the next frame call's ops; frames in flight are not affected
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_hold_lane(mc_handle* h, int lane, int hold) try {
    if (!h) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    h->hold[(size_t)lane] = hold != 0;
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_set_lane_params(mc_handle* h, int lane, const mc_lane_params* lp) try {
    if (!h) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    h->n_lane_lp += (lp != nullptr) - (h->lane_lp_set[(size_t)lane] != 0);
    h->lane_lp_set[(size_t)lane] = lp != nullptr;
    if (lp) h->lane_lp[(size_t)lane] = *lp;   // taken into the next frame call; frames in flight are not affected
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_set_lane_roi(mc_handle* h, int lane, const float* roi) try {
    if (!h) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    h->n_lane_roi += (roi != nullptr) - (h->lane_roi_set[(size_t)lane] != 0);
    h->lane_roi_set[(size_t)lane] = roi != nullptr;
    if (roi) std::copy(roi, roi + 4, h->lane_roi[(size_t)lane].begin());   // taken into the next frame call or submit
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_save_lane(mc_handle* h, int lane, void* dst, size_t cap, size_t* bytes) try {
    if (!h || !bytes) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    if (!h->inflight.empty()) { h->err = "mc_save_lane with pipelined frames in flight"; return MC_ERR_INVALID; }
    CK(cudaSetDevice(h->device));
    LaneBlob b;
    std::memset(&b, 0, sizeof(b));
    std::memcpy(b.magic, kBlobMagic, sizeof(b.magic));
    b.version = kBlobVersion;
    b.has_state = h->has_state[(size_t)lane] != 0;
    b.mode = h->t_mode; b.levels = h->t_levels; b.w = h->t_w; b.h = h->t_h; b.channels = h->t_channels;
    b.pre_down = h->t_down; b.pre_roi = h->t_roi;
    std::copy(h->t_lroi[(size_t)lane].begin(), h->t_lroi[(size_t)lane].end(), b.roi);   // the lane's own fingerprint
    if (b.has_state) {
        if (b.mode == MC_MODE_LAPLACE) {
            b.faithful = h->motion.faithful;
            b.ab_bounded = h->motion.ab_bounded;
        } else if (b.mode == MC_MODE_COLOR) {
            b.count = h->color.count[(size_t)lane]; b.head = h->color.head[(size_t)lane]; b.mod = h->color.mod[(size_t)lane];
        } else if (b.mode == MC_MODE_PHASE && h->riesz.allocated) {
            std::memcpy(b.design, &h->riesz.design[(size_t)lane], sizeof(b.design));
        }
    }
    std::vector<LanePlane> planes;
    const size_t total = lane_planes(h, b, lane, planes);
    b.bytes = sizeof(b) + total;
    *bytes = b.bytes;
    if (!dst) return MC_OK;
    if (cap < b.bytes) { h->err = "mc_save_lane: cap is smaller than the blob"; return MC_ERR_INVALID; }
    std::memcpy(dst, &b, sizeof(b));
    return copy_lane_planes(h, planes, total, (uint8_t*)dst + sizeof(b), true);
} catch (...) { return on_exception(h); }

mc_status mc_load_lane(mc_handle* h, int lane, const void* src, size_t bytes) try {
    if (!h || !src) return MC_ERR_INVALID;
    if (lane < 0 || lane >= h->lanes) { h->err = "lane out of range"; return MC_ERR_INVALID; }
    if (!h->inflight.empty()) { h->err = "mc_load_lane with pipelined frames in flight"; return MC_ERR_INVALID; }
    LaneBlob b;
    if (bytes < sizeof(b)) { h->err = "lane blob truncated"; return MC_ERR_INVALID; }
    std::memcpy(&b, src, sizeof(b));
    if (std::memcmp(b.magic, kBlobMagic, sizeof(b.magic)) != 0 || b.version != kBlobVersion) {
        h->err = "not a lane blob of this version";
        return MC_ERR_INVALID;
    }
    if (b.bytes != bytes) { h->err = "lane blob size differs from its header (truncated?)"; return MC_ERR_INVALID; }
    // the rule of single-lane restarts (color_lane_check), for the mode the lane has after the load
    auto color_refused = [&](int mode) {
        if (mode != MC_MODE_COLOR || h->lanes == 1 || h->opt.color_lane_lifecycle) return false;
        h->err = "Color mode loads one lane of a multi-lane handle only with option color_lane_lifecycle";
        return true;
    };
    CK(cudaSetDevice(h->device));
    if (!b.has_state) return color_refused(h->t_mode) ? MC_ERR_UNSUPPORTED : mc_restart_lane(h, lane);
    const bool mode_ok = b.mode == MC_MODE_LAPLACE || b.mode == MC_MODE_PHASE || b.mode == MC_MODE_COLOR;
    if (!mode_ok || (b.channels != 1 && b.channels != 3) || b.w <= 0 || b.h <= 0 || b.levels < 1 ||
        b.levels > calculate_max_levels(b.w, b.h) ||
        (b.mode == MC_MODE_COLOR && (b.mod < 2 || b.count < 1 || b.count > b.mod || b.head < 0 || b.head >= b.mod ||
                                     (b.head != 0 && b.count != b.mod)))) {
        h->err = "lane blob: bad key or window";
        return MC_ERR_INVALID;
    }
    const mc_params key = blob_key(b);
    const Roi key_roi = roi_of(key);
    const bool fresh = h->t_mode == MC_MODE_NONE;   // the handle holds no state: the load takes the blob's key
    if (!fresh && (tracker_changes(h, &key, b.levels, b.channels, b.w, b.h) || roi_differs(key_roi, h->t_lroi[(size_t)lane]))) {
        h->err = "lane blob: its key (mode, levels, size, channels, preprocess) differs from the lane's state";
        return MC_ERR_INVALID;
    }
    if (b.mode == MC_MODE_LAPLACE && ((b.faithful != 0) != h->opt.faithful_level0 ||
                                      (h->motion.allocated && h->motion.faithful != (b.faithful != 0)))) {
        h->err = "lane blob: faithful_level0 differs from the handle's";
        return MC_ERR_INVALID;
    }
    if (color_refused(b.mode)) return MC_ERR_UNSUPPORTED;
    Options opt = h->opt;
    if (opt.profile_kernels) opt.lane_groups = 1;
    const ModeCtx ctx{.stream = h->stream, .tables = &h->tables, .launches = &h->launches, .err = &h->err, .opt = opt,
                      .float_out = nullptr, .prof = nullptr};
    // The mode's state for the key, allocated as a frame call allocates it (every other lane then has no state).  An
    // allocation made here is undone when the blob turns out not to fit it.
    bool allocated_here = false;
    mc_status st = MC_OK;
    const std::vector<Roi> lroi = h->t_lroi;
    if (fresh) {   // every lane takes the blob's fingerprint (the others have no state)
        tracker_set(h, &key, b.levels, b.channels, b.w, b.h);
        h->t_lroi.assign((size_t)h->lanes, key_roi);
    }
    if (b.mode == MC_MODE_LAPLACE && !h->motion.allocated) {
        allocated_here = true;
        st = h->motion.allocate(ctx, b.w, b.h, b.channels, b.levels);
    } else if (b.mode == MC_MODE_PHASE && b.channels == 3 && !h->riesz.allocated) {
        allocated_here = true;
        st = h->riesz.allocate(ctx, b.w, b.h, nullptr, b.levels);
    } else if (b.mode == MC_MODE_COLOR && !h->color.allocated) {
        allocated_here = true;
        st = h->color.allocate(ctx, b.w, b.h, b.channels, b.levels);
    }
    std::vector<LanePlane> planes;
    const size_t total = st == MC_OK ? lane_planes(h, b, lane, planes) : 0;
    if (st != MC_OK || sizeof(b) + total != b.bytes) {
        if (allocated_here) {
            h->motion.reset(); h->riesz.reset(); h->color.reset();   // nothing else was allocated (a fresh or unallocated mode)
        }
        if (fresh) {
            tracker_disable(h);
            h->t_lroi = lroi;
        }
        if (st == MC_OK) { h->err = "lane blob size does not match its key"; st = MC_ERR_INVALID; }
        return st;
    }
    // From here a failure is a CUDA error: the state may be half-written, so it is dropped as after a failed frame.
    if (b.mode == MC_MODE_COLOR) {
        st = h->color.reserve_ring(ctx, b.mod);
        if (st == MC_OK) lane_planes(h, b, lane, planes);   // the ring may have moved
    }
    if (st == MC_OK) st = copy_lane_planes(h, planes, total, (uint8_t*)src + sizeof(b), false);
    if (st != MC_OK) {
        reset_modes(h);
        tracker_reset(h);
        return st;
    }
    if (b.mode == MC_MODE_LAPLACE) {
        h->motion.empty = false;
        h->motion.ab_bounded = h->motion.ab_bounded && b.ab_bounded;   // an unbounded state must not run L-only synthesis
    } else if (b.mode == MC_MODE_PHASE && h->riesz.allocated) {
        std::memcpy(&h->riesz.design[(size_t)lane], b.design, sizeof(b.design));
    } else if (b.mode == MC_MODE_COLOR) {
        h->color.count[(size_t)lane] = b.count; h->color.head[(size_t)lane] = b.head; h->color.mod[(size_t)lane] = b.mod;
    }
    h->has_state[(size_t)lane] = 1;
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_lane_produced(mc_handle* h, uint8_t* produced, int n) try {
    if (!h || !produced) return MC_ERR_INVALID;
    if (n != h->lanes) { h->err = "n must equal the handle's lanes"; return MC_ERR_INVALID; }
    std::memcpy(produced, h->lane_produced.data(), (size_t)n);
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_set_option(mc_handle* h, const char* key, int value) try {
    if (!h || !key) return MC_ERR_INVALID;
    Options& o = h->opt;
    if (!std::strcmp(key, "faithful_level0")) { o.faithful_level0 = value != 0; return MC_OK; }
    if (!std::strcmp(key, "keep_float_output")) { o.keep_float_output = value != 0; return MC_OK; }
    if (!std::strcmp(key, "profile_kernels")) { o.profile_kernels = value != 0; return MC_OK; }
    if (!std::strcmp(key, "use_tma")) { o.use_tma = value != 0; return MC_OK; }
    if (!std::strcmp(key, "lane_groups")) { o.lane_groups = value < 0 ? 0 : value; return MC_OK; }
    if (!std::strcmp(key, "egress_strip")) { o.egress_strip = value != 0; return MC_OK; }
    if (!std::strcmp(key, "band_from_state")) { o.band_from_state = value != 0; return MC_OK; }
    if (!std::strcmp(key, "analysis_only")) { o.analysis_only = value != 0; return MC_OK; }
    if (!std::strcmp(key, "color_lane_lifecycle")) { o.color_lane_lifecycle = value != 0; return MC_OK; }
    if (!std::strcmp(key, "pipeline_depth")) {
        if (value < 1 || value > 16 || !h->inflight.empty()) { h->err = "bad pipeline_depth"; return MC_ERR_INVALID; }
        h->depth = value;
        free_slots(h);
        return MC_OK;
    }
    h->err = std::string("unknown option ") + key;
    return MC_ERR_INVALID;
} catch (...) { return on_exception(h); }

void* mc_stream(mc_handle* h) { return h ? (void*)h->stream : nullptr; }
uint64_t mc_launch_count(mc_handle* h) { return h ? h->launches : 0; }
int mc_pipeline_depth(mc_handle* h) { return h ? h->depth : 0; }

const char* mc_last_error(mc_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

mc_status mc_sync(mc_handle* h) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_process_device(mc_handle* h, const uint8_t* d_in, int width, int height, int channels, size_t in_step,
                            const mc_params* p, uint8_t* d_out, size_t out_step, int* produced) try {
    if (!h || !produced) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return process_device_impl(h, d_in, width, height, channels, in_step, p, d_out, out_step, produced, h->lane_produced.data());
} catch (...) { return on_exception(h); }

// submit with the destination known up front: when `in`/`out` are pinned (cudaHostAlloc /
// cudaHostRegister) the copies go straight between the caller's buffers and HBM (no staging memcpy).
mc_status mc_submit(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                    const mc_params* p, uint8_t* out, size_t out_step) try {
    if (!h || !p) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    if ((int)h->inflight.size() >= h->depth) { h->err = "pipeline full: call mc_collect first"; return MC_ERR_INVALID; }
    const bool have = in != nullptr && width > 0 && height > 0 && (channels == 1 || channels == 3);
    if (have && in_step < (size_t)width * channels) { h->err = "step too small"; return MC_ERR_INVALID; }
    const Planes none;
    return submit_impl(h, have ? bgr_planes(in, width, height, channels, in_step) : none,
                       {have ? bgr_planes(out, width, height, channels, out_step) : none, none},
                       [&](const Planes& d_in, const Planes* d_out, int* produced, uint8_t* lane_produced, std::vector<uint8_t>* written) {
                           const mc_status st = process_device_impl(h, d_in.base[0], width, height, channels, d_in.pitch[0], p,
                                                                    d_out[0].base[0], d_out[0].pitch[0], produced, lane_produced);
                           std::copy(lane_produced, lane_produced + h->lanes, written[0].begin());
                           return st;
                       });
} catch (...) { return on_exception(h); }

mc_status mc_collect(mc_handle* h, int* produced) try {
    if (!h || !produced) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    if (h->inflight.empty()) { h->err = "nothing in flight"; return MC_ERR_INVALID; }
    const int si = h->inflight.front();
    h->inflight.pop_front();
    Slot& s = h->slots[(size_t)si];
    CK(cudaEventSynchronize(s.ev_done));
    *produced = s.produced;
    const size_t vl = s.lane_produced.size();   // a clip's last frame gives mc_lane_produced
    std::copy(s.lane_produced.end() - h->lanes, s.lane_produced.end(), h->lane_produced.begin());
    if (s.flags_out) std::memcpy(s.flags_out, s.lane_produced.data(), vl);
    for (int k = 0; k < kOutSets; ++k) {
        if (s.direct_out[k] || !s.out[k].base[0]) continue;
        const Planes staged = s.out[k].packed(s.h_out.p + s.out_ofs[k]);
        for (size_t l = 0; l < vl; ++l)
            if (s.written[k][l]) host_copy(s.out[k], staged, l);
    }
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_process(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                     const mc_params* p, uint8_t* out, size_t out_step, int* produced) try {
    if (!h || !produced) return MC_ERR_INVALID;
    *produced = 0;
    if (!h->inflight.empty()) { h->err = "mc_process called with pipelined frames in flight"; return MC_ERR_INVALID; }
    mc_status st = mc_submit(h, in, width, height, channels, in_step, p, out, out_step);
    if (st != MC_OK) return st;
    return mc_collect(h, produced);
} catch (...) { return on_exception(h); }

mc_status mc_state_dims(mc_handle* h, const char* name, int level, int* rows, int* cols, int* channels) try {
    if (!h || !name || !rows || !cols || !channels) return MC_ERR_INVALID;
    *rows = *cols = *channels = 0;
    StateRef r;
    if (h->t_mode == MC_MODE_LAPLACE) h->motion.find_state(name, level, r);
    else if (h->t_mode == MC_MODE_COLOR) h->color.find_state(name, level, r);
    else if (h->t_mode == MC_MODE_PHASE) h->riesz.find_state(name, level, r);
    if (r.found()) { *rows = r.rows; *cols = r.cols; *channels = r.channels; }
    return MC_OK;
} catch (...) { return on_exception(h); }

static mc_status state_xfer(mc_handle* h, const char* name, int level, float* host, size_t n, bool get) try {
    if (!h || !name || !host) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    StateRef r;
    if (h->t_mode == MC_MODE_LAPLACE) h->motion.find_state(name, level, r);
    else if (h->t_mode == MC_MODE_COLOR) h->color.find_state(name, level, r);
    else if (h->t_mode == MC_MODE_PHASE) h->riesz.find_state(name, level, r);
    if (!r.found()) { h->err = std::string("no such state: ") + name; return MC_ERR_INVALID; }
    if ((r.ptr16 || r.read_only) && !get) { h->err = std::string("read-only state: ") + name; return MC_ERR_INVALID; }
    const size_t planes = (size_t)h->lanes * r.channels;
    if (n < planes * r.rows * r.cols) { h->err = "state buffer too small"; return MC_ERR_INVALID; }
    CK(cudaStreamSynchronize(h->stream));
    // Laplace EMA state written from outside is not known to be bounded: L-only synthesis stays off until every lane's state is
    // dropped (DESIGN §4)
    if (!get && h->t_mode == MC_MODE_LAPLACE && std::strncmp(name, "lowpass", 7) == 0) h->motion.ab_bounded = false;
    if (r.ptr16) {   // int16 planes: download, then widen (exact)
        std::vector<int16_t> tmp((size_t)r.rows * r.cols);
        for (size_t pl = 0; pl < planes; ++pl) {
            CK(cudaMemcpy2D(tmp.data(), (size_t)r.cols * 2, r.ptr16 + pl * r.plane_stride, (size_t)r.pitch * 2, (size_t)r.cols * 2, r.rows,
                            cudaMemcpyDeviceToHost));
            std::copy(tmp.begin(), tmp.end(), host + pl * (size_t)r.rows * r.cols);
        }
        return MC_OK;
    }
    for (size_t pl = 0; pl < planes; ++pl) {
        const size_t lane = pl / (size_t)r.channels;
        float* d = r.lane_off.empty() ? r.ptr + pl * r.plane_stride
                                      : r.ptr + r.lane_off[lane] + (pl - lane * (size_t)r.channels) * r.plane_stride;
        float* hp = host + pl * (size_t)r.rows * r.cols;
        if (get) CK(cudaMemcpy2D(hp, (size_t)r.cols * 4, d, (size_t)r.pitch * 4, (size_t)r.cols * 4, r.rows, cudaMemcpyDeviceToHost));
        else CK(cudaMemcpy2D(d, (size_t)r.pitch * 4, hp, (size_t)r.cols * 4, (size_t)r.cols * 4, r.rows, cudaMemcpyHostToDevice));
    }
    return MC_OK;
} catch (...) { return on_exception(h); }

mc_status mc_get_state(mc_handle* h, const char* name, int level, float* dst, size_t n) try {
    return state_xfer(h, name, level, dst, n, true);
} catch (...) { return on_exception(h); }
mc_status mc_set_state(mc_handle* h, const char* name, int level, const float* src, size_t n) try {
    return state_xfer(h, name, level, const_cast<float*>(src), n, false);
} catch (...) { return on_exception(h); }

mc_status mc_get_float_output(mc_handle* h, float* dst, size_t n) try {
    if (!h || !dst) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    if (!h->float_out.p || n < h->float_out.n) { h->err = "no float output kept (set keep_float_output) or buffer too small"; return MC_ERR_INVALID; }
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(dst, h->float_out.p, h->float_out.n * sizeof(float), cudaMemcpyDeviceToHost));
    return MC_OK;
} catch (...) { return on_exception(h); }

}  // extern "C"

extern "C" void* mc_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
extern "C" void mc_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

extern "C" mc_status mc_profile_read(mc_handle* h, char* buf, size_t cap) try {
    if (!h || !buf || cap == 0) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    struct Acc { std::string name; int level; int n; double ms; };
    std::vector<Acc> acc;
    for (auto& r : h->prof.recs) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, r.a, r.b);
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
        bool found = false;
        for (auto& a : acc)
            if (a.level == r.level && a.name == r.name) { a.n++; a.ms += ms; found = true; break; }
        if (!found) acc.push_back(Acc{r.name, r.level, 1, ms});
    }
    h->prof.recs.clear();
    std::string out;
    char line[160];
    for (auto& a : acc) {
        std::snprintf(line, sizeof(line), "%s %d %d %.6f\n", a.name.c_str(), a.level, a.n, a.ms);
        out += line;
    }
    if (out.size() + 1 > cap) { h->err = "profile buffer too small"; return MC_ERR_INVALID; }
    std::memcpy(buf, out.c_str(), out.size() + 1);
    return MC_OK;
} catch (...) { return on_exception(h); }

// ---- clips: `frames` consecutive frames of every lane in one call ----------------------------------------------------
namespace {
// The argument errors of a clip call, before anything changes.  A blocking or device clip call (not `submitted`) also
// refuses while pipelined frames are in flight.
mc_status check_clip(mc_handle* h, int frames, const uint8_t* produced, bool submitted = false) {
    if (frames < 1) { h->err = "frames must be >= 1"; return MC_ERR_INVALID; }
    // frames * lanes * channels becomes a grid.z extent of the batched ingest / egress
    if ((long long)frames * h->lanes > MC_MAX_LANES) { h->err = "frames * lanes exceeds MC_MAX_LANES"; return MC_ERR_INVALID; }
    if (!produced) { h->err = "produced is null"; return MC_ERR_INVALID; }
    if (!submitted && !h->inflight.empty()) { h->err = "clip called with pipelined frames in flight"; return MC_ERR_INVALID; }
    return MC_OK;
}

// The magnifier over `frames` consecutive frames of every lane, once the clip's arguments are checked.  d_in null: the
// identity (no frame produces; a handle that was magnifying drops its state)
mc_status clip_run(mc_handle* h, const uint8_t* d_in, int frames, int w, int hh, int channels, size_t in_step, const mc_params* p,
                   uint8_t* d_out, size_t out_step, uint8_t* produced) {
    const size_t lanes = (size_t)h->lanes;
    std::fill(produced, produced + (size_t)frames * lanes, (uint8_t)0);
    int any = 0;
    mc_status st = MC_OK;
    if (p && (p->mode == MC_MODE_LAPLACE || p->mode == MC_MODE_PHASE || p->mode == MC_MODE_COLOR) && frames > 1) {
        st = process_device_impl(h, d_in, w, hh, channels, in_step, p, d_out, out_step, &any, produced, frames);
    } else {
        // one frame, and mode None: the frame path, one call per frame
        const size_t in_frame = in_step * (size_t)hh * lanes, out_frame = out_step * (size_t)hh * lanes;
        for (int t = 0; t < frames && st == MC_OK; ++t)
            st = process_device_impl(h, d_in ? d_in + (size_t)t * in_frame : nullptr, w, hh, channels, in_step, p,
                                     d_out ? d_out + (size_t)t * out_frame : nullptr, out_step, &any, produced + (size_t)t * lanes);
    }
    if (st != MC_OK) std::fill(produced, produced + (size_t)frames * lanes, (uint8_t)0);   // the state was dropped
    return st;
}

// A device clip call: checked, run, and its last frame's flags are mc_lane_produced's.
mc_status clip_impl(mc_handle* h, const uint8_t* d_in, int frames, int w, int hh, int channels, size_t in_step, const mc_params* p,
                    uint8_t* d_out, size_t out_step, uint8_t* produced) {
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    st = clip_run(h, d_in, frames, w, hh, channels, in_step, p, d_out, out_step, produced);
    std::memcpy(h->lane_produced.data(), produced + (size_t)(frames - 1) * h->lanes, (size_t)h->lanes);
    return st;
}
}  // namespace

extern "C" mc_status mc_process_clip_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                            size_t in_step, const mc_params* p, uint8_t* d_out, size_t out_step, uint8_t* produced) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return clip_impl(h, d_in, frames, width, height, channels, in_step, p, d_out, out_step, produced);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_process_clip(mc_handle* h, const uint8_t* in, int frames, int width, int height, int channels,
                                     size_t in_step, const mc_params* p, uint8_t* out, size_t out_step, uint8_t* produced) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    if (!(in != nullptr && width > 0 && height > 0 && (channels == 1 || channels == 3)))
        return clip_impl(h, nullptr, frames, 0, 0, channels, 0, p, nullptr, 0, produced);   // the identity
    const Planes src = bgr_planes(in, width, height, channels, in_step), dst = bgr_planes(out, width, height, channels, out_step);
    if (in_step < src.row[0] || (out && out_step < src.row[0])) { h->err = "step too small"; return MC_ERR_INVALID; }
    const size_t vl = (size_t)frames * h->lanes;
    CK(h->k_in.grow(src.lane_bytes() * vl));
    CK(h->k_out.grow(src.lane_bytes() * vl));
    const Planes d_in = src.packed(h->k_in.p), d_out = src.packed(h->k_out.p);
    if ((st = copy_planes(h, d_in, src, 0, vl, cudaMemcpyHostToDevice, h->stream)) != MC_OK) return st;
    st = clip_impl(h, d_in.base[0], frames, width, height, channels, d_in.pitch[0], p, d_out.base[0], d_out.pitch[0], produced);
    if (st != MC_OK) return st;
    // only the frames that produced are downloaded, one copy per run of consecutive ones ([t][lane] order); the bytes of
    // the others in `out` are left as they are
    if (out)
        st = for_each_run(vl, [&](size_t i) { return produced[i] != 0; }, [&](size_t a, size_t b) {
            return copy_planes(h, dst, d_out, a, b, cudaMemcpyDeviceToHost, h->stream);
        });
    if (st != MC_OK) return st;
    CK(cudaStreamSynchronize(h->stream));
    return MC_OK;
} catch (...) { return on_exception(h); }

// ---- NV12 frames: converted into BGR staging, magnified as BGR, converted back into the caller's planes ---------------
namespace {
mc_status check_nv12(mc_handle* h, std::initializer_list<const mc_nv12*> frame_sets, int w, int hh, int vlanes, const mc_params* p) {
    if (!p) { h->err = "params is null"; return MC_ERR_INVALID; }
    for (const mc_nv12* f : frame_sets) {
        if (const char* e = Source::nv12(f, w, hh).check((size_t)vlanes)) { h->err = e; return MC_ERR_INVALID; }
    }
    return MC_OK;
}

Nv12Planes planes_of(const mc_nv12& f) { return Nv12Planes{f.y, f.uv, f.uv + 1, f.pitch, f.pitch, f.lane_stride, kNv12ChromaStep}; }

// Row pitch of the BGR staging: 16-byte rows keep the conversions on their 64-bit path.
size_t bgr_step_of(int w) { return (size_t)round_up(3 * w, 16); }

// One kernel launch of the handle's own (`launch()` issues it on the handle's stream): counted, and timed as `name` under
// profile_kernels.
template <class Launch>
mc_status launch_counted(mc_handle* h, const char* name, Launch launch) {
    const bool prof = h->opt.profile_kernels && h->prof.begin(name, 0, h->stream);
    const cudaError_t e = launch();
    if (prof) h->prof.end(h->stream);
    CK(e);
    ++h->launches;
    return MC_OK;
}

// `in` (NV12 or I420) -> h->n_in (BGR, bgr_step_of(w)) for `vlanes` virtual lanes, and h->n_out sized for the magnifier's
// BGR output unless the caller writes it elsewhere (bgr_out false).  Mode None does not read its input: no launch.
mc_status nv12_ingest(mc_handle* h, const Nv12Planes& in, int w, int hh, int vlanes, const mc_params* p, bool bgr_out = true) {
    const size_t bytes = bgr_step_of(w) * hh * vlanes;
    CK(h->n_in.grow(bytes));
    if (bgr_out) CK(h->n_out.grow(bytes));
    if (p->mode == MC_MODE_NONE) return MC_OK;
    return launch_counted(h, "nv12_to_bgr", [&] {
        return launch_nv12_to_bgr(in, w, hh, vlanes, h->n_in.p, bgr_step_of(w), h->stream);
    });
}

// h->n_out -> `out` for the virtual lanes whose flag (host, vlanes bytes) is set.  When only some produced, the flags go
// to the device on the handle's stream, as the modes upload their lane ops: no host synchronisation.
mc_status nv12_egress(mc_handle* h, const mc_nv12& out, int w, int hh, int vlanes, const uint8_t* flags) {
    const int n = (int)std::count_if(flags, flags + vlanes, [](uint8_t f) { return f != 0; });
    if (n == 0) return MC_OK;
    const uint8_t* d_flags = nullptr;
    if (n < vlanes) {
        CK(h->n_flags.grow((size_t)vlanes));
        CK(cudaMemcpyAsync(h->n_flags.p, flags, (size_t)vlanes, cudaMemcpyHostToDevice, h->stream));
        d_flags = h->n_flags.p;
    }
    return launch_counted(h, "bgr_to_nv12", [&] {
        return launch_bgr_to_nv12(h->n_out.p, bgr_step_of(w), w, hh, vlanes, d_flags, out.y, out.uv, out.pitch, out.lane_stride,
                                  h->stream);
    });
}

// One frame call on NV12 device planes: nv12_ingest -> the magnifier on the BGR staging -> nv12_egress.
mc_status nv12_frame(mc_handle* h, const mc_nv12& in, const mc_nv12& out, int w, int hh, const mc_params* p, int* produced,
                     uint8_t* lane_produced) {
    mc_status st = nv12_ingest(h, planes_of(in), w, hh, h->lanes, p);
    if (st != MC_OK) return st;
    const size_t step = bgr_step_of(w);
    if ((st = process_device_impl(h, h->n_in.p, w, hh, 3, step, p, h->n_out.p, step, produced, lane_produced)) != MC_OK) return st;
    return nv12_egress(h, out, w, hh, h->lanes, lane_produced);
}
}  // namespace

extern "C" mc_status mc_process_nv12_device(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p,
                                            const mc_nv12* out, int* produced) try {
    if (!h || !produced) return MC_ERR_INVALID;
    *produced = 0;
    CK(cudaSetDevice(h->device));
    const mc_status st = check_nv12(h, {in, out}, width, height, h->lanes, p);
    if (st != MC_OK) return st;
    return nv12_frame(h, *in, *out, width, height, p, produced, h->lane_produced.data());
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_process_clip_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                                 const mc_params* p, const mc_nv12* out, uint8_t* produced) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    const int vlanes = frames * h->lanes;
    if ((st = check_nv12(h, {in, out}, width, height, vlanes, p)) != MC_OK) return st;
    if ((st = nv12_ingest(h, planes_of(*in), width, height, vlanes, p)) != MC_OK) return st;
    const size_t step = bgr_step_of(width);
    st = clip_impl(h, h->n_in.p, frames, width, height, 3, step, p, h->n_out.p, step, produced);
    if (st != MC_OK) return st;
    return nv12_egress(h, *out, width, height, vlanes, produced);
} catch (...) { return on_exception(h); }

// mc_submit on NV12 planes: the slot buffers hold NV12, so PCIe moves 1.5 B/px each way; the conversions run on the
// compute stream around the magnifier, through the handle's BGR staging (stream-ordered, shared by the slots).
extern "C" mc_status mc_submit_nv12(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p,
                                    const mc_nv12* out) try {
    if (!h || !p) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    if ((int)h->inflight.size() >= h->depth) { h->err = "pipeline full: call mc_collect first"; return MC_ERR_INVALID; }
    const mc_status st = check_nv12(h, {in, out}, width, height, h->lanes, p);
    if (st != MC_OK) return st;
    return submit_impl(h, nv12_planes(*in, width, height), {nv12_planes(*out, width, height), Planes{}},
                       [&](const Planes& d_in, const Planes* d_out, int* produced, uint8_t* lane_produced, std::vector<uint8_t>* written) {
                           const mc_status st = nv12_frame(h, nv12_of(d_in), nv12_of(d_out[0]), width, height, p, produced,
                                                           lane_produced);
                           std::copy(lane_produced, lane_produced + h->lanes, written[0].begin());
                           return st;
                       });
} catch (...) { return on_exception(h); }

// ---- the processing chain: runChainOnce (ChainBuilder.cpp:19-29) = Preprocess -> Grayscale -> Magnification ----------
namespace {
// What runChainOnce does to a w x hh x channels frame before the magnifier.
struct ChainGeom {
    bool pre = false, gray = false;                       // PreprocessProcessor crops / downscales; GrayscaleProcessor converts
    int rx = 0, ry = 0, rw = 0, rh = 0;                   // the ROI in the frame
    int dw = 0, dh = 0, cc = 0;                           // the magnifier's input: size and channels
    int kind = FRONT_COPY, isx = 1, isy = 1;              // how the ROI becomes dw x dh
    std::vector<int2> org;                                // per lane: its own ROI origin (mc_set_lane_roi); empty: rx, ry
    bool front() const { return pre || gray; }
};

// PreprocessProcessor.cpp:10-51 and GrayscaleProcessor.cpp:7-16 as geometry, and the info of a frame the magnifier does not
// produce.  -> an error text, or null.
const char* chain_geometry(const mc_params* p, int w, int hh, int channels, int grayscale, ChainGeom& g, mc_chain_info* info) {
    std::memset(info, 0, sizeof(*info));
    info->cur_is_input = 1; info->orig_is_input = 1;
    g = ChainGeom{};
    if (w <= 0 || hh <= 0) return nullptr;   // empty image: every stage is an identity (PreprocessProcessor.cpp:11)
    if (channels != 1 && channels != 3) return "channels must be 1 or 3";
    const int divisor = std::min(std::max((int)p->pre_downscale, 1), 8);
    g.pre = p->pre_roiEnabled != 0 || divisor != 1;
    g.gray = grayscale != 0 && channels == 3;
    g.cc = g.gray ? 1 : channels;
    g.rw = g.dw = w; g.rh = g.dh = hh;
    if (g.pre) {
        preprocess_roi(w, hh, p->pre_roiEnabled != 0, p->pre_roiX, p->pre_roiY, p->pre_roiW, p->pre_roiH, g.rx, g.ry, g.rw, g.rh);
        g.dw = g.rw; g.dh = g.rh;
        if (divisor > 1) {   // cv::resize(INTER_AREA); integer scales on both axes take OpenCV's "area fast" path
            g.dw = std::max(1, g.rw / divisor); g.dh = std::max(1, g.rh / divisor);
            const double sx = (double)g.rw / g.dw, sy = (double)g.rh / g.dh;
            g.isx = (int)sx; g.isy = (int)sy;
            const double eps = 2.220446049250313e-16;   // DBL_EPSILON
            g.kind = std::abs(sx - g.isx) < eps && std::abs(sy - g.isy) < eps ? FRONT_AREA_FAST : FRONT_AREA;
        }
        info->orig_is_input = 0; info->orig_w = g.dw; info->orig_h = g.dh; info->orig_channels = channels;
    }
    if (g.front()) { info->cur_is_input = 0; info->out_w = g.dw; info->out_h = g.dh; info->out_channels = g.cc; }
    return nullptr;
}

// chain_geometry of a call on the handle's lanes, each cropped at its effective ROI (mc_set_lane_roi).  The first lane
// that runs (lane 0 when every lane is held) gives the geometry and the info; every other running lane must crop a
// rectangle of the same pixel size, which then starts at the lane's own origin (g.org, left empty when every origin is
// (g.rx, g.ry)).  Held lanes are not cropped, so they are checked when they run again.
mc_status chain_lane_geometry(mc_handle* h, const mc_params* p, int w, int hh, int channels, int grayscale, ChainGeom& g,
                              mc_chain_info* info) {
    const size_t lanes = (size_t)h->lanes;
    size_t first = 0;
    while (first < lanes && h->hold[first]) ++first;
    if (first == lanes) first = 0;
    mc_params q = *p;
    const Roi r0 = lane_roi(h, *p, first);
    q.pre_roiX = r0[0]; q.pre_roiY = r0[1]; q.pre_roiW = r0[2]; q.pre_roiH = r0[3];
    if (const char* e = chain_geometry(&q, w, hh, channels, grayscale, g, info)) { h->err = e; return MC_ERR_INVALID; }
    if (!g.pre || !p->pre_roiEnabled || h->n_lane_roi == 0) return MC_OK;
    std::vector<int2> org(lanes, make_int2(g.rx, g.ry));
    bool same = true;
    for (size_t l = 0; l < lanes; ++l) {
        if (h->hold[l]) continue;
        const Roi r = lane_roi(h, *p, l);
        int x, y, rw, rh;
        preprocess_roi(w, hh, true, r[0], r[1], r[2], r[3], x, y, rw, rh);
        if (rw != g.rw || rh != g.rh) {
            h->err = "lane " + std::to_string(l) + "'s ROI crops " + std::to_string(rw) + "x" + std::to_string(rh) + ", lane " +
                     std::to_string(first) + "'s " + std::to_string(g.rw) + "x" + std::to_string(g.rh) +
                     ": the lanes of a call must crop rectangles of one size";
            return MC_ERR_INVALID;
        }
        org[l] = make_int2(x, y);
        same = same && x == g.rx && y == g.ry;
    }
    if (!same) g.org = std::move(org);
    return MC_OK;
}

// The general INTER_AREA tap tables of g on the device, in one buffer (x taps, y taps, x offsets, y offsets): built and
// uploaded on the handle's stream only when (rw, dw, rh, dh) changes.
mc_status area_tables(mc_handle* h, const ChainGeom& g, FrontArgs& a) {
    const int key[4] = {g.rw, g.dw, g.rh, g.dh};
    if (!std::equal(key, key + 4, h->f_tab_key)) {
        std::fill(h->f_tab_key, h->f_tab_key + 4, -1);
        std::vector<AreaTap> xt, yt;
        std::vector<int> xo, yo;
        build_area_tab(g.rw, g.dw, (double)g.rw / g.dw, xt, xo);
        build_area_tab(g.rh, g.dh, (double)g.rh / g.dh, yt, yo);
        const size_t bx = xt.size() * sizeof(AreaTap), by = yt.size() * sizeof(AreaTap), bxo = xo.size() * sizeof(int);
        const size_t total = bx + by + bxo + yo.size() * sizeof(int);
        std::vector<uint8_t>& b = h->f_tabs_host;   // lives on the handle: the copy is asynchronous
        b.resize(total);
        std::memcpy(b.data(), xt.data(), bx);
        std::memcpy(b.data() + bx, yt.data(), by);
        std::memcpy(b.data() + bx + by, xo.data(), bxo);
        std::memcpy(b.data() + bx + by + bxo, yo.data(), total - bx - by - bxo);
        CK(h->f_tabs.grow(total));
        CK(cudaMemcpyAsync(h->f_tabs.p, b.data(), total, cudaMemcpyHostToDevice, h->stream));
        h->f_tab_ofs[0] = bx; h->f_tab_ofs[1] = bx + by; h->f_tab_ofs[2] = bx + by + bxo;
        std::copy(key, key + 4, h->f_tab_key);
    }
    const uint8_t* t = h->f_tabs.p;
    a.xtab = (const AreaTap*)t;
    a.ytab = (const AreaTap*)(t + h->f_tab_ofs[0]);
    a.xofs = (const int*)(t + h->f_tab_ofs[1]);
    a.yofs = (const int*)(t + h->f_tab_ofs[2]);
    return MC_OK;
}

// compose(): each pane is the chain's output cropped to its even size; the canvas holds one or two panes.
void canvas_size(const ChainGeom& g, int split, int& cw, int& ch) {
    const int w = g.dw & ~1, hh = g.dh & ~1;
    cw = ch = 0;
    if (w <= 0 || hh <= 0) return;   // Exporter.cpp:57, 64: an empty pane, no frame
    cw = split == MC_SPLIT_LEFT_RIGHT ? 2 * w : w;
    ch = split == MC_SPLIT_TOP_BOTTOM ? 2 * hh : hh;
}

// A chain call's export canvas (mc_chain_compose_device): the split and where the canvases go.
struct ComposeReq {
    int split;
    const mc_canvas* canvas;
};

const char* check_compose(const ComposeReq& c, const ChainGeom& g, size_t vl, const mc_handle::Overlay& ov) {
    if (c.split < MC_SPLIT_NONE || c.split > MC_SPLIT_TOP_BOTTOM) return "split out of range";
    const mc_canvas* cv = c.canvas;
    if (!cv || cv->format < MC_CANVAS_BGR || cv->format > MC_CANVAS_RGB_PLANAR) return "canvas is null or of an unknown format";
    const bool yuv420 = cv->format == MC_CANVAS_NV12 || cv->format == MC_CANVAS_I420;
    if (!cv->data || (yuv420 && !cv->uv)) return "canvas plane is null";
    if (cv->format == MC_CANVAS_I420 && cv->pitch % 2) return "I420 canvas pitch is odd";
    int cw, ch;
    canvas_size(g, c.split, cw, ch);
    if (ov.set && cw > 0 && (cw != ov.cw || ch != ov.ch)) return "canvas geometry differs from the overlay's";
    if (cv->pitch < (size_t)cw * (cv->format == MC_CANVAS_BGR || cv->format == MC_CANVAS_RGB ? 3 : 1))
        return "canvas pitch < canvas row";
    const size_t planes = cv->format == MC_CANVAS_RGB_PLANAR ? 3 : 1;
    if (vl > 1 && cv->lane_stride < planes * cv->pitch * ch) return "canvas lane_stride < pitch * canvas height (per plane)";
    return nullptr;
}

// Where a chain call's results go: the processed frames and the original tap (null: not wanted), or with cmp the export
// canvases instead.
struct ChainDst {
    uint8_t* out = nullptr; size_t out_step = 0;     // the processed frames
    uint8_t* orig = nullptr; size_t orig_step = 0;   // the original tap
    std::optional<ComposeReq> cmp;
};

// The argument errors of a chain call on `frames` consecutive frames of every lane, before anything changes, and its
// geometry g and info.  Only the pointers' nullness is read, so host and device frame sets are checked alike.
// out_optional: a NULL d.out is not an error.
mc_status chain_check(mc_handle* h, const Source& s, int frames, const mc_params* p, int grayscale, const ChainDst& d,
                      mc_chain_info* info, ChainGeom& g, bool out_optional = false) {
    if (!p || !info) { h->err = "params or info is null"; return MC_ERR_INVALID; }
    const bool empty = s.empty();
    mc_status st = chain_lane_geometry(h, p, empty ? 0 : s.w, empty ? 0 : s.hh, s.channels, grayscale, g, info);
    if (st != MC_OK) return st;
    const bool pre = g.pre || s.converts(), front = g.front() || s.converts();
    const size_t lanes = (size_t)h->lanes, vl = (size_t)frames * lanes;
    if (s.converts()) {   // info says where the conversion went; the frame's errors come before the canvas's
        info->orig_is_input = 0; info->orig_w = g.dw; info->orig_h = g.dh; info->orig_channels = 3;
        info->cur_is_input = 0; info->out_w = g.dw; info->out_h = g.dh; info->out_channels = g.cc;
        if (const char* e = s.check(vl)) { h->err = e; return MC_ERR_INVALID; }
    }
    if (d.cmp) {
        if (const char* e = check_compose(*d.cmp, g, vl, h->ov)) { h->err = e; return MC_ERR_INVALID; }
    }
    if (empty) return MC_OK;   // the identity
    if (const char* e = s.converts() ? nullptr : s.check(vl)) { h->err = e; return MC_ERR_INVALID; }
    if (p->mode < 0 || p->mode > MC_MODE_NONE) { h->err = "bad mode"; return MC_ERR_INVALID; }
    if (!d.cmp && (front || p->mode != MC_MODE_NONE)) {
        if (!d.out && !out_optional) { h->err = "output pointer is null"; return MC_ERR_INVALID; }
        if (d.out_step < (size_t)g.dw * g.cc) { h->err = "out_step too small"; return MC_ERR_INVALID; }
    }
    if (!d.cmp && pre && d.orig && d.orig_step < (size_t)g.dw * s.channels) {
        h->err = "original_step too small";
        return MC_ERR_INVALID;
    }
    const int max_levels = calculate_max_levels(g.dw, g.dh);
    if (p->mode == MC_MODE_COLOR && max_levels >= 1 && !(lanes == 1 && h->hold[0])) {
        const int levels = std::min(std::max((int)p->levels, 1), max_levels);
        return color_lane_check(h, p, levels, g.cc, g.dw, g.dh);
    }
    return MC_OK;
}

// runChainOnce for every lane and `frames` consecutive frames, on device frame sets that passed chain_check (which gave
// g).  One front launch writes the preprocessed frames (d.orig, or staging) and the magnifier's input (the same frames or
// their gray), the magnifier writes d.out, and the frames it did not produce get the front's output.  produced: frames *
// lanes flags.  With d.cmp, the call composes instead: the magnifier writes h->x_mag, the preprocessed frames stay in
// h->f_pre when the canvas shows them, and one compose launch reads every pane where it is.
// Everything it uses of the handle's chain scratch (f_pre, f_gray, f_flags, f_tabs, n_in, x_mag, x_ops and the host
// copies) is written and read on the handle's stream only, so pipelined frames may share it in submit order.
mc_status chain_run(mc_handle* h, const ChainGeom& g, const Source& s, int frames, const mc_params* p, ChainDst d, uint8_t* produced) {
    const size_t lanes = (size_t)h->lanes, vl = (size_t)frames * lanes;
    if (s.empty()) return clip_run(h, nullptr, frames, 0, 0, s.channels, 0, p, nullptr, 0, produced);
    const bool pre = g.pre || s.converts(), front = g.front() || s.converts();
    const size_t out_row = (size_t)g.dw * g.cc;
    mc_status st;
    if (d.cmp) {
        if (p->mode != MC_MODE_NONE) {
            CK(h->x_mag.grow(out_row * g.dh * vl));
            d.out = h->x_mag.p; d.out_step = out_row;
        }
        d.orig = nullptr;
        if ((g.pre || s.composes_from_tap()) && d.cmp->split != MC_SPLIT_NONE) {
            d.orig_step = (size_t)g.dw * s.channels;
            CK(h->f_pre.grow(d.orig_step * g.dh * vl));
            d.orig = h->f_pre.p;
        }
    }
    const bool tap = pre && d.orig;
    // ---- the front: one launch over the virtual lanes; held lanes are skipped
    const PaneSrc input = s.pane();
    const uint8_t* mag_in = input.p;
    size_t mag_step = input.step;
    if (front) {
        FrontArgs a;
        a.src = input.p; a.step = input.step; a.lane_stride = input.lane_stride;
        a.cb = input.cb; a.cr = input.cr; a.cpitch = input.cpitch; a.cstep = input.cstep;
        a.rx = g.rx; a.ry = g.ry; a.dw = g.dw; a.dh = g.dh; a.kind = g.kind; a.isx = g.isx; a.isy = g.isy;
        if (tap) {
            a.dst = d.orig; a.dst_step = d.orig_step;
        } else if (pre && !g.gray) {   // the preprocessed frames are the magnifier's input
            a.dst_step = (size_t)g.dw * s.channels;
            CK(h->f_pre.grow(a.dst_step * g.dh * vl));
            a.dst = h->f_pre.p;
        }
        a.dst_lane_stride = a.dst_step * g.dh;
        if (g.gray) {
            CK(h->f_gray.grow((size_t)g.dw * g.dh * vl));
            a.gray = h->f_gray.p;
        }
        if (g.kind == FRONT_AREA && (st = area_tables(h, g, a)) != MC_OK) return st;
        if (!g.org.empty()) {   // the lanes' own crop origins go up on the handle's stream, as the held-lane flags do
            h->f_org_host.resize(vl);   // lives on the handle: the copy is asynchronous
            for (size_t v = 0; v < vl; ++v) h->f_org_host[v] = g.org[v % lanes];
            CK(h->f_org.grow(vl));
            CK(cudaMemcpyAsync(h->f_org.p, h->f_org_host.data(), vl * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
            a.org = h->f_org.p;
        }
        if (std::any_of(h->hold.begin(), h->hold.end(), [](uint8_t x) { return x != 0; })) {
            h->f_flags_host.resize(vl);   // lives on the handle: the copy is asynchronous
            for (size_t v = 0; v < vl; ++v) h->f_flags_host[v] = !h->hold[v % lanes];
            CK(h->f_flags.grow(vl));
            CK(cudaMemcpyAsync(h->f_flags.p, h->f_flags_host.data(), vl, cudaMemcpyHostToDevice, h->stream));
            a.flags = h->f_flags.p;
        }
        if ((st = launch_counted(h, "chain_front", [&] { return launch_chain_front(a, input.kind, (int)vl, h->stream); })) != MC_OK) return st;
        mag_in = g.gray ? a.gray : a.dst;
        mag_step = g.gray ? (size_t)g.dw : a.dst_step;
    } else if (!s.bgr_or_gray() && p->mode != MC_MODE_NONE) {   // 4:2:0 without a front stage: a plain 4:2:0 -> BGR conversion
        if ((st = nv12_ingest(h, yuv420_of(s.planes), s.w, s.hh, (int)vl, p, false)) != MC_OK) return st;
        mag_in = h->n_in.p;
        mag_step = bgr_step_of(s.w);
    }

    // ---- the magnifier, straight into d.out; then the canvases, or the front's output for the frames it did not produce
    if ((st = clip_run(h, mag_in, frames, g.dw, g.dh, g.cc, mag_step, p, d.out, d.out_step, produced)) != MC_OK) return st;
    if (d.cmp) {
        ComposeArgs a;
        a.w = g.dw & ~1; a.h = g.dh & ~1;
        if (a.w <= 0 || a.h <= 0) return MC_OK;   // a 0 x 0 canvas
        const int in_kind = s.channels == 3 ? FRONT_BGR : FRONT_GRAY, out_kind = g.cc == 3 ? FRONT_BGR : FRONT_GRAY;
        a.src[0] = tap ? PaneSrc{d.orig, nullptr, d.orig_step, d.orig_step * g.dh, in_kind} : input;
        a.src[1] = PaneSrc{d.out, nullptr, d.out_step, d.out_step * g.dh, out_kind};
        a.src[2] = front ? PaneSrc{mag_in, nullptr, mag_step, mag_step * g.dh, out_kind} : input;
        // the pane choice of every virtual lane goes to the device on the handle's stream, as the front's flags do
        h->x_ops_host.resize(vl);   // lives on the handle: the copy is asynchronous
        for (size_t v = 0; v < vl; ++v)
            h->x_ops_host[v] = h->hold[v % lanes] ? COMPOSE_SKIP : produced[v] ? COMPOSE_MAGNIFIED : COMPOSE_FALLBACK;
        CK(h->x_ops.grow(vl));
        CK(cudaMemcpyAsync(h->x_ops.p, h->x_ops_host.data(), vl, cudaMemcpyHostToDevice, h->stream));
        a.ops = h->x_ops.p;
        a.split = d.cmp->split;
        const mc_canvas& cv = *d.cmp->canvas;
        a.format = cv.format;
        a.data = cv.data; a.uv = cv.uv; a.pitch = cv.pitch; a.lane_stride = cv.lane_stride;
        int cw, ch;
        canvas_size(g, a.split, cw, ch);
        if (cv.format == MC_CANVAS_I420) {   // the Cr plane follows the Cb plane's canvas_h / 2 rows of pitch / 2 bytes
            a.cr = cv.uv + cv.pitch / 2 * (size_t)(ch / 2);
        } else if (cv.format == MC_CANVAS_RGB_PLANAR) {   // the G and B planes follow the R plane's canvas_h rows
            a.uv = cv.data + cv.pitch * (size_t)ch;
            a.cr = cv.data + 2 * cv.pitch * (size_t)ch;
        }
        if (h->ov.set) {
            a.ov_rects = h->ov.rects;
            a.ov_map = h->ov_dev.p;
            for (int i = 0; i < h->ov.rects; ++i) {
                a.ov[i] = h->ov.rect[i];
                a.ov[i].index = reinterpret_cast<const uint16_t*>(h->ov_dev.p + h->ov.ofs[i]);
            }
        }
        return launch_counted(h, "compose", [&] { return launch_compose(a, (int)vl, h->stream); });
    }
    if (!front) return MC_OK;
    const size_t in_lane = mag_step * g.dh, out_lane = d.out_step * g.dh;
    return for_each_run(vl, [&](size_t v) { return !produced[v] && !h->hold[v % lanes]; }, [&](size_t a, size_t b) -> mc_status {
        CK(cudaMemcpy2DAsync(d.out + a * out_lane, d.out_step, mag_in + a * in_lane, mag_step, out_row, (b - a) * g.dh,
                             cudaMemcpyDeviceToDevice, h->stream));
        return MC_OK;
    });
}

// A device chain call: checked (with the pipelined frames' refusal), run, and its last frame's flags are
// mc_lane_produced's.
mc_status chain_impl(mc_handle* h, const Source& s, int frames, const mc_params* p, int grayscale, const ChainDst& d,
                     uint8_t* produced, mc_chain_info* info) {
    if (s.missing) { h->err = s.missing; return MC_ERR_INVALID; }
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    ChainGeom g;
    if ((st = chain_check(h, s, frames, p, grayscale, d, info, g)) != MC_OK) return st;
    if ((st = chain_run(h, g, s, frames, p, d, produced)) != MC_OK) return st;
    const size_t lanes = (size_t)h->lanes, vl = (size_t)frames * lanes;
    std::memcpy(h->lane_produced.data(), produced + vl - lanes, lanes);
    info->magnified = std::any_of(produced, produced + vl, [](uint8_t x) { return x != 0; });
    return MC_OK;
}
}  // namespace

extern "C" mc_status mc_chain_geometry(const mc_params* p, int width, int height, int channels, int grayscale,
                                       mc_chain_info* info) try {
    if (!p || !info) return MC_ERR_INVALID;
    ChainGeom g;
    return chain_geometry(p, width, height, channels, grayscale, g, info) ? MC_ERR_INVALID : MC_OK;
} catch (...) { return on_exception(nullptr); }

extern "C" mc_status mc_chain_process_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                             size_t in_step, const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                             uint8_t* d_original, size_t original_step, uint8_t* produced,
                                             mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::bgr(d_in, width, height, channels, in_step), frames, p, grayscale,
                      ChainDst{d_out, out_step, d_original, original_step}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_process_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                                  const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                                  uint8_t* d_original, size_t original_step, uint8_t* produced,
                                                  mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::nv12(in, width, height), frames, p, grayscale, ChainDst{d_out, out_step, d_original, original_step},
                      produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_compose_geometry(const mc_params* p, int width, int height, int channels, int grayscale, int split,
                                         int* canvas_w, int* canvas_h) try {
    if (!p || !canvas_w || !canvas_h || split < MC_SPLIT_NONE || split > MC_SPLIT_TOP_BOTTOM) return MC_ERR_INVALID;
    ChainGeom g;
    mc_chain_info info;
    if (chain_geometry(p, width, height, channels, grayscale, g, &info)) return MC_ERR_INVALID;
    canvas_size(g, split, *canvas_w, *canvas_h);
    return MC_OK;
} catch (...) { return on_exception(nullptr); }

namespace {
const char* check_overlay(const mc_overlay& o) {
    static_assert(kOverlayRects == MC_OVERLAY_MAX_RECTS, "the kernel's rect count is the ABI's");
    if (o.canvas_w < 1 || o.canvas_h < 1) return "overlay canvas size < 1";
    if (o.rects < 0 || o.rects > MC_OVERLAY_MAX_RECTS) return "overlay rects out of range";
    if (o.maps < 1 || o.maps > 65536 || !o.map) return "overlay maps out of range or map is null";
    for (int i = 0; i < o.rects; ++i) {
        const mc_overlay_rect& r = o.rect[i];
        if (!r.index) return "overlay index is null";
        if (r.w < 1 || r.h < 1 || r.x < 0 || r.y < 0 || r.x > o.canvas_w - r.w || r.y > o.canvas_h - r.h)
            return "overlay rect is empty or not inside the canvas";
        for (int j = 0; j < i; ++j) {
            const mc_overlay_rect& q = o.rect[j];
            if (r.x < q.x + q.w && q.x < r.x + r.w && r.y < q.y + q.h && q.y < r.y + r.h) return "overlay rects overlap";
        }
        const size_t n = (size_t)r.w * r.h;
        if (std::any_of(r.index, r.index + n, [&](uint16_t m) { return m >= o.maps; })) return "overlay index >= maps";
    }
    return nullptr;
}
}  // namespace

extern "C" mc_status mc_set_overlay(mc_handle* h, const mc_overlay* o) try {
    if (!h) return MC_ERR_INVALID;
    if (!o) { h->ov.set = false; return MC_OK; }
    if (const char* e = check_overlay(*o)) { h->err = e; return MC_ERR_INVALID; }
    CK(cudaSetDevice(h->device));
    // one host image of maps and index planes, uploaded in one copy on the handle's stream: compose launches enqueued
    // before it still read the previous overlay.  The source is pageable, so it is staged before the call returns.
    mc_handle::Overlay ov;
    ov.cw = o->canvas_w; ov.ch = o->canvas_h; ov.rects = o->rects;
    size_t total = (size_t)o->maps * 256;
    for (int i = 0; i < o->rects; ++i) {
        const mc_overlay_rect& r = o->rect[i];
        ov.rect[i] = OverlayRect{r.x, r.y, r.w, r.h, nullptr};
        ov.ofs[i] = total;
        total += (size_t)r.w * r.h * sizeof(uint16_t);
    }
    std::vector<uint8_t>& b = h->ov_host;
    b.resize(total);
    std::memcpy(b.data(), o->map, (size_t)o->maps * 256);
    for (int i = 0; i < o->rects; ++i)
        std::memcpy(b.data() + ov.ofs[i], o->rect[i].index, (size_t)o->rect[i].w * o->rect[i].h * sizeof(uint16_t));
    h->ov.set = false;   // a CUDA error from here on leaves no overlay (and says so)
    CK(h->ov_dev.grow(total));   // frees a smaller old copy first: cudaFree waits for the launches that read it
    CK(cudaMemcpyAsync(h->ov_dev.p, b.data(), total, cudaMemcpyHostToDevice, h->stream));
    ov.set = true;
    h->ov = ov;
    return MC_OK;
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                             size_t in_step, const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                             uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::bgr(d_in, width, height, channels, in_step), frames, p, grayscale,
                      ChainDst{.cmp = ComposeReq{split, canvas}}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                                  const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                  uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::nv12(in, width, height), frames, p, grayscale, ChainDst{.cmp = ComposeReq{split, canvas}}, produced,
                      info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_process_yuv422_device(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                                    const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                                    uint8_t* d_original, size_t original_step, uint8_t* produced,
                                                    mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::yuv422(in, width, height), frames, p, grayscale, ChainDst{d_out, out_step, d_original, original_step},
                      produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_yuv422_device(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                                    const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                    uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::yuv422(in, width, height), frames, p, grayscale, ChainDst{.cmp = ComposeReq{split, canvas}},
                      produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_process_yuv420p_device(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                                     const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                                     uint8_t* d_original, size_t original_step, uint8_t* produced,
                                                     mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::yuv420p(in, width, height), frames, p, grayscale,
                      ChainDst{d_out, out_step, d_original, original_step}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_yuv420p_device(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                                     const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                     uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::yuv420p(in, width, height), frames, p, grayscale, ChainDst{.cmp = ComposeReq{split, canvas}},
                      produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_process_rgb_device(mc_handle* h, const mc_rgb* in, int frames, int width, int height,
                                                 const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                                 uint8_t* d_original, size_t original_step, uint8_t* produced,
                                                 mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::rgb(in, width, height), frames, p, grayscale, ChainDst{d_out, out_step, d_original, original_step},
                      produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_rgb_device(mc_handle* h, const mc_rgb* in, int frames, int width, int height,
                                                 const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                 uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_impl(h, Source::rgb(in, width, height), frames, p, grayscale, ChainDst{.cmp = ComposeReq{split, canvas}},
                      produced, info);
} catch (...) { return on_exception(h); }

namespace {
// The body of the chain submits and of the blocking host chain calls: chain_check on the host frame set, then one slot of
// the pipeline whose run is chain_run on the slot's buffers.  The processed frames go to d.out (lane k at k * out_h *
// out_step) and the original tap to d.orig (lane k at k * orig_h * orig_step).  out_optional: a NULL d.out is not an
// error; the processed frames are then not downloaded.
mc_status chain_submit(mc_handle* h, const Source& s, const mc_params* p, int grayscale, const ChainDst& d, mc_chain_info* info,
                       bool out_optional = false) {
    if (s.missing) { h->err = s.missing; return MC_ERR_INVALID; }
    if ((int)h->inflight.size() >= h->depth) { h->err = "pipeline full: call mc_collect first"; return MC_ERR_INVALID; }
    ChainGeom g;
    mc_status st = chain_check(h, s, 1, p, grayscale, d, info, g, out_optional);
    if (st != MC_OK) return st;
    const bool empty = s.empty(), front = g.front() || s.converts(), tap = (g.pre || s.converts()) && d.orig;
    Planes src, dst[kOutSets];
    if (!empty) {
        src = s.planes;
        dst[0] = bgr_planes(d.out, g.dw, g.dh, g.cc, d.out_step);
        if (tap) dst[1] = bgr_planes(d.orig, g.dw, g.dh, s.channels, d.orig_step);
    }
    // Room for the largest outputs of this frame size (no crop or downscale, no gray), so that a ROI, downscale or grayscale
    // change with frames in flight does not have to grow the slots.
    const size_t full = empty ? 0 : ((size_t)s.w * s.hh * s.channels * h->lanes + 255) / 256 * 256;
    return submit_impl(h, src, dst, [&](const Planes& d_in, const Planes* d_out, int* produced, uint8_t* lane_produced,
                                        std::vector<uint8_t>* written) {
        const ChainDst slot{d_out[0].base[0], d_out[0].pitch[0], d_out[1].base[0], d_out[1].pitch[0]};
        const mc_status rs = chain_run(h, g, s.on(d_in), 1, p, slot, lane_produced);
        if (rs != MC_OK) return rs;
        *produced = std::any_of(lane_produced, lane_produced + h->lanes, [](uint8_t x) { return x != 0; });
        for (size_t l = 0; l < (size_t)h->lanes; ++l) {   // what chain_run wrote: see mc_chain_process_device
            written[0][l] = lane_produced[l] || (front && !h->hold[l]);
            written[1][l] = tap && !h->hold[l];
        }
        return MC_OK;
    }, d.orig ? 2 * full : full);
}

// The blocking 1-lane host calls: chain_submit + mc_collect into tight buffers.  A source that converts (4:2:2) always
// writes both frames, so a buffer too small for its frame is refused before anything runs.  A BGR or gray frame's buffer
// that turns out too small for what the chain wrote is not downloaded, and the call returns MC_ERR_INVALID once the frame
// ran.
mc_status chain_host_call(mc_handle* h, const char* name, const Source& s, const mc_params* p, int grayscale, uint8_t* out,
                          size_t out_bytes, uint8_t* original, size_t original_bytes, mc_chain_info* info) {
    std::memset(info, 0, sizeof(*info));
    info->cur_is_input = 1; info->orig_is_input = 1;
    if (h->lanes != 1) { h->err = std::string(name) + " needs a 1-lane handle"; return MC_ERR_INVALID; }
    if (!h->inflight.empty()) { h->err = std::string(name) + " called with pipelined frames in flight"; return MC_ERR_INVALID; }
    if (h->hold[0]) { h->err = std::string(name) + " called while lane 0 is held"; return MC_ERR_INVALID; }
    if (s.missing) { h->err = s.missing; return MC_ERR_INVALID; }
    ChainGeom g;
    const bool empty = s.empty();
    mc_status st = chain_lane_geometry(h, p, empty ? 0 : s.w, empty ? 0 : s.hh, s.channels, grayscale, g, info);
    if (st != MC_OK) return st;
    const size_t out_frame = (size_t)g.dw * g.dh * g.cc, orig_frame = (size_t)g.dw * g.dh * s.channels;
    const bool out_fits = out && out_bytes >= out_frame, orig_fits = original && original_bytes >= orig_frame;
    if (s.converts() && out && !out_fits) { h->err = "out buffer too small"; return MC_ERR_INVALID; }
    if (s.converts() && original && !orig_fits) { h->err = "original buffer too small"; return MC_ERR_INVALID; }
    const ChainDst tight{out_fits ? out : nullptr, (size_t)g.dw * g.cc, orig_fits ? original : nullptr, (size_t)g.dw * s.channels};
    st = chain_submit(h, s, p, grayscale, tight, info, true);
    if (st != MC_OK) return st;
    int produced = 0;
    if ((st = mc_collect(h, &produced)) != MC_OK) return st;
    info->magnified = produced != 0;
    if (produced && info->cur_is_input) {   // no front stage: the magnified frame is the chain's result
        info->cur_is_input = 0; info->out_w = g.dw; info->out_h = g.dh; info->out_channels = g.cc;
    }
    if (!info->orig_is_input && original && !orig_fits) { h->err = "original buffer too small"; return MC_ERR_INVALID; }
    if (!info->cur_is_input && out && !out_fits) { h->err = "out buffer too small"; return MC_ERR_INVALID; }
    return MC_OK;
}
}  // namespace

// The one-lane host form: the frame is uploaded, runs the device chain, and what it wrote comes back tight.
extern "C" mc_status mc_chain_process(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                                      const mc_params* p, int grayscale, uint8_t* out, size_t out_bytes, uint8_t* original,
                                      size_t original_bytes, mc_chain_info* info) try {
    if (!h || !p || !info) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_host_call(h, "mc_chain_process", Source::bgr(in, width, height, channels, in_step), p, grayscale, out, out_bytes,
                           original, original_bytes, info);
} catch (...) { return on_exception(h); }

// The live camera form: the 2 * width bytes of each row go up in one 2D copy, run the device chain, and both of its
// frames (always written for a 4:2:2 source) come back tight.  Every argument is checked before the upload.
extern "C" mc_status mc_chain_process_yuv422(mc_handle* h, const mc_yuv422* in, int width, int height, const mc_params* p,
                                             int grayscale, uint8_t* out, size_t out_bytes, uint8_t* original,
                                             size_t original_bytes, mc_chain_info* info) try {
    if (!h || !p || !info) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_host_call(h, "mc_chain_process_yuv422", Source::yuv422(in, width, height), p, grayscale, out, out_bytes, original,
                           original_bytes, info);
} catch (...) { return on_exception(h); }

// The pipelined host chain: one frame of every lane per submit, collected by mc_collect in submit order with mc_submit and
// mc_submit_nv12 frames.
extern "C" mc_status mc_chain_submit(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                                     const mc_params* p, int grayscale, uint8_t* out, size_t out_step, uint8_t* original,
                                     size_t original_step, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_submit(h, Source::bgr(in, width, height, channels, in_step), p, grayscale,
                        ChainDst{out, out_step, original, original_step}, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_submit_nv12(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p, int grayscale,
                                          uint8_t* out, size_t out_step, uint8_t* original, size_t original_step,
                                          mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_submit(h, Source::nv12(in, width, height), p, grayscale, ChainDst{out, out_step, original, original_step}, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_submit_yuv422(mc_handle* h, const mc_yuv422* in, int width, int height, const mc_params* p,
                                            int grayscale, uint8_t* out, size_t out_step, uint8_t* original, size_t original_step,
                                            mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_submit(h, Source::yuv422(in, width, height), p, grayscale, ChainDst{out, out_step, original, original_step}, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_submit_yuv420p(mc_handle* h, const mc_yuv420p* in, int width, int height, const mc_params* p,
                                             int grayscale, uint8_t* out, size_t out_step, uint8_t* original, size_t original_step,
                                             mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_submit(h, Source::yuv420p(in, width, height), p, grayscale, ChainDst{out, out_step, original, original_step},
                        info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_submit_rgb(mc_handle* h, const mc_rgb* in, int width, int height, const mc_params* p, int grayscale,
                                         uint8_t* out, size_t out_step, uint8_t* original, size_t original_step,
                                         mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return chain_submit(h, Source::rgb(in, width, height), p, grayscale, ChainDst{out, out_step, original, original_step}, info);
} catch (...) { return on_exception(h); }

// ---- the export canvas from host clips: compose submits, collected by mc_collect -----------------------------------------
namespace {
// The planes of the canvases of a cw x ch canvas geometry (BGR or RGB; NV12 luma and Cb,Cr; I420 luma, Cb and Cr; planar R,
// G and B), virtual lane v at v * lane_stride.  Only the canvas_w (chroma: canvas_w / 2) bytes of each row are copied.
Planes canvas_planes(const mc_canvas& c, int cw, int ch) {
    const size_t w = (size_t)cw, hh = (size_t)ch;
    if (c.format == MC_CANVAS_NV12) return Planes{{c.data, c.uv}, {hh, hh / 2}, {w, w}, {c.pitch, c.pitch}, c.lane_stride};
    if (c.format == MC_CANVAS_I420)
        return Planes{{c.data, c.uv, c.uv + c.pitch / 2 * (hh / 2)}, {hh, hh / 2, hh / 2}, {w, w / 2, w / 2},
                      {c.pitch, c.pitch / 2, c.pitch / 2}, c.lane_stride};
    if (c.format == MC_CANVAS_RGB_PLANAR)
        return Planes{{c.data, c.data + c.pitch * hh, c.data + 2 * c.pitch * hh}, {hh, hh, hh}, {w, w, w},
                      {c.pitch, c.pitch, c.pitch}, c.lane_stride};
    return Planes{{c.data}, {hh}, {w * 3}, {c.pitch}, c.lane_stride};
}

// The body of the compose submits: every check of the matching device compose call (without its refusal while frames are
// in flight), then one slot of the pipeline whose run is chain_run with a ComposeReq on the slot's buffers.  The compose
// kernel writes the canvases into the slot's own output, never into handle scratch that the next submit reuses, and the
// canvases of the lanes that are not held come back from there.  `produced` (frames * lanes) is written by the mc_collect
// of this submit.
mc_status compose_submit(mc_handle* h, const Source& s, int frames, const mc_params* p, int grayscale, const ComposeReq& cmp,
                         uint8_t* produced, mc_chain_info* info) {
    if (s.missing) { h->err = s.missing; return MC_ERR_INVALID; }
    if ((int)h->inflight.size() >= h->depth) { h->err = "pipeline full: call mc_collect first"; return MC_ERR_INVALID; }
    mc_status st = check_clip(h, frames, produced, true);
    if (st != MC_OK) return st;
    ChainGeom g;
    if ((st = chain_check(h, s, frames, p, grayscale, ChainDst{.cmp = cmp}, info, g)) != MC_OK) return st;
    const bool empty = s.empty();
    // the device call's magnifier refuses Color lanes with different parameters only once its front ran: here, before any copy
    if (!empty && calculate_max_levels(g.dw, g.dh) >= 1 && (st = lane_params_check(h, *p)) != MC_OK) return st;
    int cw, ch;
    canvas_size(g, cmp.split, cw, ch);
    Planes src, dst[kOutSets];
    if (!empty) {
        src = s.planes;
        if (cw > 0) dst[0] = canvas_planes(*cmp.canvas, cw, ch);
    }
    // Room for the canvases of this frame size without a crop or downscale, so that a ROI or downscale change with clips in
    // flight does not have to grow the slots; a shorter clip fits in a longer one's.
    ChainGeom full;
    full.dw = empty ? 0 : s.w; full.dh = empty ? 0 : s.hh;
    int fw, fh;
    canvas_size(full, cmp.split, fw, fh);
    const size_t reserve =
        ((size_t)fw * fh * (cmp.canvas->format == MC_CANVAS_NV12 || cmp.canvas->format == MC_CANVAS_I420 ? 3 : 6) / 2 * frames *
             h->lanes + 255) / 256 * 256;
    const size_t lanes = (size_t)h->lanes, vl = (size_t)frames * lanes;
    return submit_impl(h, src, dst, [&](const Planes& d_in, const Planes* d_out, int* any, uint8_t* flags,
                                        std::vector<uint8_t>* written) {
        const mc_canvas slot{cmp.canvas->format, d_out[0].base[0], d_out[0].base[1], d_out[0].pitch[0], d_out[0].lane_stride};
        const mc_status rs = chain_run(h, g, s.on(d_in), frames, p, ChainDst{.cmp = ComposeReq{cmp.split, &slot}}, flags);
        if (rs != MC_OK) return rs;
        *any = std::any_of(flags, flags + vl, [](uint8_t x) { return x != 0; });
        for (size_t v = 0; v < vl; ++v) written[0][v] = cw > 0 && !h->hold[v % lanes];   // what the compose kernel wrote
        return MC_OK;
    }, reserve, frames, produced);
}
}  // namespace

// The pipelined exporter: a clip of every lane through the chain and compose per submit, collected by mc_collect in
// submit order with every other submit.
extern "C" mc_status mc_chain_compose_submit(mc_handle* h, const uint8_t* in, int frames, int width, int height, int channels,
                                             size_t in_step, const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                             uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return compose_submit(h, Source::bgr(in, width, height, channels, in_step), frames, p, grayscale, ComposeReq{split, canvas},
                          produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_submit_nv12(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                                  const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                  uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return compose_submit(h, Source::nv12(in, width, height), frames, p, grayscale, ComposeReq{split, canvas}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_submit_yuv422(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                                    const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                    uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return compose_submit(h, Source::yuv422(in, width, height), frames, p, grayscale, ComposeReq{split, canvas}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_submit_yuv420p(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                                     const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                     uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return compose_submit(h, Source::yuv420p(in, width, height), frames, p, grayscale, ComposeReq{split, canvas}, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_compose_submit_rgb(mc_handle* h, const mc_rgb* in, int frames, int width, int height,
                                                 const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                                 uint8_t* produced, mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    return compose_submit(h, Source::rgb(in, width, height), frames, p, grayscale, ComposeReq{split, canvas}, produced, info);
} catch (...) { return on_exception(h); }

/* test hooks, not declared in the public header: the two conversion kernels alone on device buffers (default stream,
 * synchronised); they return the cudaError_t */
extern "C" int mc_debug_nv12_to_bgr(const mc_nv12* in, int width, int height, int lanes, uint8_t* d_bgr, size_t bgr_step) {
    cudaError_t e = launch_nv12_to_bgr(planes_of(*in), width, height, lanes, d_bgr, bgr_step, nullptr);
    return (int)(e != cudaSuccess ? e : cudaStreamSynchronize(nullptr));
}
extern "C" int mc_debug_bgr_to_nv12(const uint8_t* d_bgr, size_t bgr_step, int width, int height, int lanes, const uint8_t* d_flags,
                                    const mc_nv12* out) {
    cudaError_t e = launch_bgr_to_nv12(d_bgr, bgr_step, width, height, lanes, d_flags, out->y, out->uv, out->pitch, out->lane_stride,
                                       nullptr);
    return (int)(e != cudaSuccess ? e : cudaStreamSynchronize(nullptr));
}
