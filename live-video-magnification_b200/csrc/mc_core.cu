// The handle behind the C ABI: an H100-resident twin of livim::MagnificationProcessor
// (reference src/processing/MagnificationProcessor.cpp:10-67) — level clamp, structural reset,
// mode dispatch, passthrough decisions — plus device memory, streams and the pinned pipeline.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <deque>
#include <initializer_list>
#include <new>
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

// A frame set: one plane per lane (BGR or gray: height rows of w * c bytes) or two (NV12: height luma rows and height / 2
// Cb,Cr rows of w bytes).  Rows hold `row` bytes and are `pitch` apart; lane l starts l * lane_stride after lane 0.
struct Planes {
    uint8_t* base[2] = {nullptr, nullptr};
    size_t rows[2] = {0, 0};   // rows per lane; 0: no second plane
    size_t row = 0, pitch = 0, lane_stride = 0;

    size_t lane_rows() const { return rows[0] + rows[1]; }
    size_t lane_bytes() const { return lane_rows() * row; }
    // the same shape packed at `p`: no row padding, the second plane right after the first, lanes back to back
    Planes packed(uint8_t* p) const { return Planes{{p, p + rows[0] * row}, {rows[0], rows[1]}, row, row, lane_bytes()}; }
    // `lanes` consecutive lanes are one run of lanes * lane_rows() rows `pitch` apart
    bool one_run(size_t lanes) const {
        return (!rows[1] || base[1] == base[0] + rows[0] * pitch) && (lanes == 1 || lane_stride == lane_rows() * pitch);
    }
};

Planes bgr_planes(const uint8_t* p, int w, int hh, int c, size_t step) {
    return Planes{{const_cast<uint8_t*>(p), nullptr}, {(size_t)hh, 0}, (size_t)w * c, step, step * hh};
}
Planes nv12_planes(const mc_nv12& f, int w, int hh) {
    return Planes{{f.y, f.uv}, {(size_t)hh, (size_t)hh / 2}, (size_t)w, f.pitch, f.lane_stride};
}
mc_nv12 nv12_of(const Planes& f) { return mc_nv12{f.base[0], f.base[1], f.pitch, f.lane_stride}; }

struct Slot {  // one in-flight frame of the pinned pipeline; frees what it holds
    uint8_t *h_in = nullptr, *h_out = nullptr;   // pinned staging (lanes frames, packed)
    DeviceBuffer<> d_in, d_out;                  // device frames (packed)
    cudaEvent_t ev_in = nullptr, ev_k = nullptr, ev_done = nullptr;
    int produced = 0;
    std::vector<uint8_t> lane_produced;          // per lane: its bytes of `out` are written
    Planes out;                                  // the caller's destination (base null: none)
    bool direct_out = false;                     // D2H went straight into `out` (pinned)
    ~Slot() {
        for (uint8_t* p : {h_in, h_out}) if (p) cudaFreeHost(p);
        for (cudaEvent_t e : {ev_in, ev_k, ev_done}) if (e) cudaEventDestroy(e);
    }
};
}  // namespace

struct mc_handle {
    int device = 0;
    int lanes = 1;
    cudaStream_t stream = nullptr, s_in = nullptr, s_out = nullptr;
    DeviceTables tables;
    std::string err;
    uint64_t launches = 0;

    // StructuralTracker (MagnifyCore.hpp:45-80)
    int t_mode = MC_MODE_NONE, t_levels = -1, t_channels = -1, t_w = 0, t_h = 0;
    int t_down = 1, t_roi = 0;
    float t_rx = 0.f, t_ry = 0.f, t_rw = 1.f, t_rh = 1.f;

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
    // mc_chain_process: device copies of its host frame, processed frame and original tap
    DeviceBuffer<> c_raw, c_out, c_orig;

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
    h->t_down = 1; h->t_roi = 0; h->t_rx = 0.f; h->t_ry = 0.f; h->t_rw = 1.f; h->t_rh = 1.f;
}
bool tracker_changes(const mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    return p->mode != h->t_mode || lv != h->t_levels || w != h->t_w || hh != h->t_h ||
           ch != h->t_channels || p->pre_downscale != h->t_down ||
           (p->pre_roiEnabled != 0) != (h->t_roi != 0) || p->pre_roiX != h->t_rx ||
           p->pre_roiY != h->t_ry || p->pre_roiW != h->t_rw || p->pre_roiH != h->t_rh;
}
bool tracker_update(mc_handle* h, const mc_params* p, int lv, int ch, int w, int hh) {
    const bool change = tracker_changes(h, p, lv, ch, w, hh);
    if (change) {
        h->t_mode = p->mode; h->t_levels = lv; h->t_w = w; h->t_h = hh; h->t_channels = ch;
        h->t_down = p->pre_downscale; h->t_roi = p->pre_roiEnabled != 0;
        h->t_rx = p->pre_roiX; h->t_ry = p->pre_roiY; h->t_rw = p->pre_roiW; h->t_rh = p->pre_roiH;
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

mc_status ensure_slots(mc_handle* h, size_t bytes) {
    if ((int)h->slots.size() == h->depth && h->slots[0].d_in.n >= bytes) return MC_OK;
    if (!h->inflight.empty()) {
        h->err = "pipeline geometry changed with frames in flight";
        return MC_ERR_INVALID;
    }
    free_slots(h);
    h->slots = std::vector<Slot>((size_t)h->depth);
    for (auto& s : h->slots) {
        s.lane_produced.assign((size_t)h->lanes, 0);
        CK(cudaHostAlloc((void**)&s.h_in, bytes, cudaHostAllocDefault));
        CK(cudaHostAlloc((void**)&s.h_out, bytes, cudaHostAllocDefault));
        CK(s.d_in.grow(bytes));
        CK(s.d_out.grow(bytes));
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
bool is_pinned(const Planes& f) { return is_pinned(f.base[0]) && (!f.rows[1] || is_pinned(f.base[1])); }

// Lane l of every plane, host to host, row by row.
void host_copy(const Planes& dst, const Planes& src, size_t l) {
    for (int k = 0; k < 2; ++k)
        for (size_t r = 0; r < src.rows[k]; ++r)
            std::memcpy(dst.base[k] + l * dst.lane_stride + r * dst.pitch, src.base[k] + l * src.lane_stride + r * src.pitch, src.row);
}

// Lanes [a, b) of every plane between host and device: one copy when both sides hold them as one run of rows (a plain
// copy when neither side pads its rows), otherwise one 2D copy per plane and lane.
mc_status copy_planes(mc_handle* h, const Planes& dst, const Planes& src, size_t a, size_t b, cudaMemcpyKind kind, cudaStream_t s) {
    if (dst.one_run(b - a) && src.one_run(b - a)) {
        uint8_t* d = dst.base[0] + a * dst.lane_stride;
        const uint8_t* from = src.base[0] + a * src.lane_stride;
        const size_t rows = (b - a) * src.lane_rows();
        if (dst.pitch == src.row && src.pitch == src.row) CK(cudaMemcpyAsync(d, from, rows * src.row, kind, s));
        else CK(cudaMemcpy2DAsync(d, dst.pitch, from, src.pitch, src.row, rows, kind, s));
        return MC_OK;
    }
    for (size_t l = a; l < b; ++l)
        for (int k = 0; k < 2; ++k)
            if (src.rows[k])
                CK(cudaMemcpy2DAsync(dst.base[k] + l * dst.lane_stride, dst.pitch, src.base[k] + l * src.lane_stride, src.pitch, src.row,
                                     src.rows[k], kind, s));
    return MC_OK;
}

// Without option "color_lane_lifecycle" a multi-lane Color handle keeps its lanes in lock-step: a frame call while a lane
// is held, or restarted while others run, is MC_ERR_UNSUPPORTED, checked before any state changes.
mc_status color_lane_check(mc_handle* h, const mc_params* p, int levels, int channels, int w, int hh) {
    if (h->opt.color_lane_lifecycle) return MC_OK;
    const bool change = tracker_changes(h, p, levels, channels, w, hh);
    int n_hold = 0, n_state = 0;
    for (int l = 0; l < h->lanes; ++l) { n_hold += h->hold[(size_t)l] != 0; n_state += h->has_state[(size_t)l] != 0; }
    if (n_hold) { h->err = "Color mode cannot hold a lane of a multi-lane handle"; return MC_ERR_UNSUPPORTED; }
    if (!change && n_state != 0 && n_state != h->lanes) {
        h->err = "Color mode cannot restart one lane of a multi-lane handle while the others run";
        return MC_ERR_UNSUPPORTED;
    }
    return MC_OK;
}

// The body of MagnificationProcessor::process on device-resident frames.
// lane_produced: `lanes` per-lane flags (written).  frames > 1 (Laplace and Phase): a clip of that many consecutive
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
    Options opt = h->opt;
    if (opt.profile_kernels) opt.lane_groups = 1;   // one launch chain: the events time one kernel at a time
    const ModeCtx ctx{.stream = h->stream, .tables = &h->tables, .launches = &h->launches, .err = &h->err, .opt = opt,
                      .float_out = opt.keep_float_output ? h->float_out.p : nullptr,
                      .prof = opt.profile_kernels ? &h->prof : nullptr,
                      .lane_ops = h->ops.data(), .d_lane_ops = h->d_ops, .lane_produced = lane_produced, .held_lost = &held_lost};
    mc_status st = MC_OK;
    switch (p->mode) {
        case MC_MODE_LAPLACE: st = h->motion.process(ctx, io, *p, levels, produced, frames); break;
        case MC_MODE_COLOR: st = h->color.process(ctx, io, *p, levels, produced); break;
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
        else if (held_lost) h->has_state[(size_t)l] = 0;
    }
    return st;
}

// One frame set into the pipeline.  `in` is uploaded on the input stream into the next slot's packed device copy:
// directly when it is pinned, through the slot's pinned staging when not.  `run(d_in, d_out, produced, lane_produced)`
// then fills the slot's packed output on the handle's stream (with no buffers when `in` is empty: the identity).  Only
// the lanes that produced are downloaded on the output stream, one copy per run of consecutive ones, into `out` when it
// is pinned and into the staging, which mc_collect copies out, when not; the other lanes' bytes of `out` stay as they
// are.  The slot's d_in is not overwritten before its kernels ran: the next upload into it follows mc_collect of this
// frame, which waits on ev_done.
template <class Run>
mc_status submit_impl(mc_handle* h, const Planes& in, const Planes& out, Run run) {
    const size_t lanes = (size_t)h->lanes, bytes = in.lane_bytes() * lanes;
    mc_status st = ensure_slots(h, std::max<size_t>(bytes, 1));
    if (st != MC_OK) return st;
    if (out.base[0] && out.pitch < out.row) { h->err = "out_step too small"; return MC_ERR_INVALID; }
    const int si = h->next_slot;
    Slot& s = h->slots[(size_t)si];
    s.produced = 0; s.out = out; s.direct_out = false;
    const Planes none, d_in = bytes ? in.packed(s.d_in.p) : none, d_out = bytes ? in.packed(s.d_out.p) : none;
    if (bytes) {
        const bool pinned = is_pinned(in);
        const Planes src = pinned ? in : in.packed(s.h_in);
        if (!pinned)
            for (size_t l = 0; l < lanes; ++l) host_copy(src, in, l);
        if ((st = copy_planes(h, d_in, src, 0, lanes, cudaMemcpyHostToDevice, h->s_in)) != MC_OK) return st;
        CK(cudaEventRecord(s.ev_in, h->s_in));
        CK(cudaStreamWaitEvent(h->stream, s.ev_in, 0));
    }
    int produced = 0;
    if ((st = run(d_in, d_out, &produced, s.lane_produced.data())) != MC_OK) return st;
    s.produced = produced;
    if (produced) {
        CK(cudaEventRecord(s.ev_k, h->stream));
        CK(cudaStreamWaitEvent(h->s_out, s.ev_k, 0));
        if (out.base[0]) {
            s.direct_out = is_pinned(out);
            const Planes dst = s.direct_out ? out : out.packed(s.h_out);
            st = for_each_run(lanes, [&](size_t l) { return s.lane_produced[l] != 0; }, [&](size_t a, size_t b) {
                return copy_planes(h, dst, d_out, a, b, cudaMemcpyDeviceToHost, h->s_out);
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
    if (lut.empty()) { g_create_error = "embedded Lab LUT missing"; mc_destroy(h); return MC_ERR_INVALID; }
    std::vector<float4> gam;
    build_inv_gamma_spline(gam);
    build_lab_inv_coeffs(h->tables.inv_coeffs);
    if ((e = cudaMalloc((void**)&h->tables.lab_lut, lut.size() * sizeof(LabLutCell))) != cudaSuccess) return fail("cudaMalloc lut", e);
    if ((e = cudaMalloc((void**)&h->tables.inv_gamma, gam.size() * sizeof(float4))) != cudaSuccess) return fail("cudaMalloc gamma", e);
    if ((e = cudaMemcpy(h->tables.lab_lut, lut.data(), lut.size() * sizeof(LabLutCell), cudaMemcpyHostToDevice)) != cudaSuccess) return fail("copy lut", e);
    if ((e = cudaMemcpy(h->tables.inv_gamma, gam.data(), gam.size() * sizeof(float4), cudaMemcpyHostToDevice)) != cudaSuccess) return fail("copy gamma", e);
    h->motion.lanes = h->color.lanes = h->riesz.lanes = lanes;
    h->has_state.assign((size_t)lanes, 0);
    h->hold.assign((size_t)lanes, 0);
    h->ops.assign((size_t)lanes, 0);
    h->lane_produced.assign((size_t)lanes, 0);
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
    if (!std::strcmp(key, "prefetch_state")) { o.prefetch_state = value != 0; return MC_OK; }
    if (!std::strcmp(key, "lane_groups")) { o.lane_groups = value < 0 ? 0 : value; return MC_OK; }
    if (!std::strcmp(key, "egress_strip")) { o.egress_strip = value == 1 ? 16 : value; return MC_OK; }
    if (!std::strcmp(key, "ingest_warps")) { o.ingest_warps = value; return MC_OK; }
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
                       have ? bgr_planes(out, width, height, channels, out_step) : none,
                       [&](const Planes& d_in, const Planes& d_out, int* produced, uint8_t* lane_produced) {
                           return process_device_impl(h, d_in.base[0], width, height, channels, d_in.pitch, p, d_out.base[0],
                                                      d_out.pitch, produced, lane_produced);
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
    h->lane_produced = s.lane_produced;
    if (s.produced && !s.direct_out && s.out.base[0]) {
        const Planes staged = s.out.packed(s.h_out);
        for (size_t l = 0; l < (size_t)h->lanes; ++l)
            if (s.lane_produced[l]) host_copy(s.out, staged, l);
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
    if (r.ptr16 && !get) { h->err = std::string("read-only state: ") + name; return MC_ERR_INVALID; }
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
        float* d = r.ptr + pl * r.plane_stride;
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
// The argument errors of a clip call, before anything changes.
mc_status check_clip(mc_handle* h, int frames, const uint8_t* produced) {
    if (frames < 1) { h->err = "frames must be >= 1"; return MC_ERR_INVALID; }
    // frames * lanes * channels becomes a grid.z extent of the batched ingest / egress
    if ((long long)frames * h->lanes > MC_MAX_LANES) { h->err = "frames * lanes exceeds MC_MAX_LANES"; return MC_ERR_INVALID; }
    if (!produced) { h->err = "produced is null"; return MC_ERR_INVALID; }
    if (!h->inflight.empty()) { h->err = "clip called with pipelined frames in flight"; return MC_ERR_INVALID; }
    return MC_OK;
}

// d_in null: the identity (no frame produces; a handle that was magnifying drops its state)
mc_status clip_impl(mc_handle* h, const uint8_t* d_in, int frames, int w, int hh, int channels, size_t in_step, const mc_params* p,
                    uint8_t* d_out, size_t out_step, uint8_t* produced) {
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    const size_t lanes = (size_t)h->lanes;
    std::fill(produced, produced + (size_t)frames * lanes, (uint8_t)0);
    int any = 0;
    if (p && (p->mode == MC_MODE_LAPLACE || p->mode == MC_MODE_PHASE) && frames > 1) {
        st = process_device_impl(h, d_in, w, hh, channels, in_step, p, d_out, out_step, &any, produced, frames);
    } else {
        // Color (and every mode with one frame): the frame path, one call per frame
        const size_t in_frame = in_step * (size_t)hh * lanes, out_frame = out_step * (size_t)hh * lanes;
        for (int t = 0; t < frames && st == MC_OK; ++t)
            st = process_device_impl(h, d_in ? d_in + (size_t)t * in_frame : nullptr, w, hh, channels, in_step, p,
                                     d_out ? d_out + (size_t)t * out_frame : nullptr, out_step, &any, produced + (size_t)t * lanes);
    }
    if (st != MC_OK) std::fill(produced, produced + (size_t)frames * lanes, (uint8_t)0);   // the state was dropped
    std::memcpy(h->lane_produced.data(), produced + (size_t)(frames - 1) * lanes, lanes);
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
    if (in_step < src.row || (out && out_step < src.row)) { h->err = "step too small"; return MC_ERR_INVALID; }
    const size_t vl = (size_t)frames * h->lanes;
    CK(h->k_in.grow(src.lane_bytes() * vl));
    CK(h->k_out.grow(src.lane_bytes() * vl));
    const Planes d_in = src.packed(h->k_in.p), d_out = src.packed(h->k_out.p);
    if ((st = copy_planes(h, d_in, src, 0, vl, cudaMemcpyHostToDevice, h->stream)) != MC_OK) return st;
    st = clip_impl(h, d_in.base[0], frames, width, height, channels, d_in.pitch, p, d_out.base[0], d_out.pitch, produced);
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
    if (w < 2 || hh < 2 || (w & 1) || (hh & 1)) { h->err = "NV12 width and height must be even and >= 2"; return MC_ERR_INVALID; }
    for (const mc_nv12* f : frame_sets) {
        if (!f || !f->y || !f->uv) { h->err = "NV12 plane is null"; return MC_ERR_INVALID; }
        if (f->pitch < (size_t)w) { h->err = "NV12 pitch < width"; return MC_ERR_INVALID; }
        if (vlanes > 1 && f->lane_stride < f->pitch * hh) { h->err = "NV12 lane_stride < pitch * height"; return MC_ERR_INVALID; }
    }
    return MC_OK;
}

Nv12Planes planes_of(const mc_nv12& f) { return Nv12Planes{f.y, f.uv, f.pitch, f.lane_stride}; }

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

// `in` -> h->n_in (BGR, bgr_step_of(w)) for `vlanes` virtual lanes, and h->n_out sized for the magnifier's BGR output
// unless the caller writes it elsewhere (bgr_out false).  Mode None does not read its input: no launch.
mc_status nv12_ingest(mc_handle* h, const mc_nv12& in, int w, int hh, int vlanes, const mc_params* p, bool bgr_out = true) {
    const size_t bytes = bgr_step_of(w) * hh * vlanes;
    CK(h->n_in.grow(bytes));
    if (bgr_out) CK(h->n_out.grow(bytes));
    if (p->mode == MC_MODE_NONE) return MC_OK;
    return launch_counted(h, "nv12_to_bgr", [&] {
        return launch_nv12_to_bgr(planes_of(in), w, hh, vlanes, h->n_in.p, bgr_step_of(w), h->stream);
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
    mc_status st = nv12_ingest(h, in, w, hh, h->lanes, p);
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
    if ((st = nv12_ingest(h, *in, width, height, vlanes, p)) != MC_OK) return st;
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
    return submit_impl(h, nv12_planes(*in, width, height), nv12_planes(*out, width, height),
                       [&](const Planes& d_in, const Planes& d_out, int* produced, uint8_t* lane_produced) {
                           return nv12_frame(h, nv12_of(d_in), nv12_of(d_out), width, height, p, produced, lane_produced);
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

// runChainOnce for every lane and `frames` consecutive frames: the source is d_in (u8 BGR or gray, in_step) or, when nv
// is not null, NV12 planes (channels 3).  Everything is checked before the front kernel runs; then one front launch
// writes the preprocessed frames (d_original, or staging) and the magnifier's input (the same frames or their gray),
// the magnifier writes d_out, and the frames it did not produce get the front's output.  produced: frames * lanes flags.
mc_status chain_impl(mc_handle* h, const uint8_t* d_in, size_t in_step, const mc_nv12* nv, int frames, int w, int hh,
                     int channels, const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step, uint8_t* d_orig,
                     size_t orig_step, uint8_t* produced, mc_chain_info* info) {
    if (!p || !info) { h->err = "params or info is null"; return MC_ERR_INVALID; }
    const bool empty = !nv && (d_in == nullptr || w <= 0 || hh <= 0);
    ChainGeom g;
    if (const char* e = chain_geometry(p, empty ? 0 : w, empty ? 0 : hh, channels, grayscale, g, info)) {
        h->err = e;
        return MC_ERR_INVALID;
    }
    mc_status st = check_clip(h, frames, produced);
    if (st != MC_OK) return st;
    if (empty) return clip_impl(h, nullptr, frames, 0, 0, channels, 0, p, nullptr, 0, produced);   // the identity
    const size_t lanes = (size_t)h->lanes, vl = (size_t)frames * lanes;
    if (nv) {
        if ((st = check_nv12(h, {nv}, w, hh, (int)vl, p)) != MC_OK) return st;
    } else if (in_step < (size_t)w * channels) {
        h->err = "step too small";
        return MC_ERR_INVALID;
    }
    if (p->mode < 0 || p->mode > MC_MODE_NONE) { h->err = "bad mode"; return MC_ERR_INVALID; }
    const size_t out_row = (size_t)g.dw * g.cc;
    if (g.front() || p->mode != MC_MODE_NONE) {
        if (!d_out) { h->err = "output pointer is null"; return MC_ERR_INVALID; }
        if (out_step < out_row) { h->err = "out_step too small"; return MC_ERR_INVALID; }
    }
    const bool tap = g.pre && d_orig;
    if (tap && orig_step < (size_t)g.dw * channels) { h->err = "original_step too small"; return MC_ERR_INVALID; }
    const int max_levels = calculate_max_levels(g.dw, g.dh);
    if (p->mode == MC_MODE_COLOR && max_levels >= 1 && !(lanes == 1 && h->hold[0])) {
        const int levels = std::min(std::max((int)p->levels, 1), max_levels);
        if ((st = color_lane_check(h, p, levels, g.cc, g.dw, g.dh)) != MC_OK) return st;
    }

    // ---- the front: one launch over the virtual lanes; held lanes are skipped
    const uint8_t* mag_in = d_in;
    size_t mag_step = in_step;
    if (g.front()) {
        FrontArgs a;
        if (nv) { a.src = nv->y; a.uv = nv->uv; a.step = nv->pitch; a.lane_stride = nv->lane_stride; }
        else { a.src = d_in; a.step = in_step; a.lane_stride = in_step * hh; }
        a.rx = g.rx; a.ry = g.ry; a.dw = g.dw; a.dh = g.dh; a.kind = g.kind; a.isx = g.isx; a.isy = g.isy;
        if (tap) {
            a.dst = d_orig; a.dst_step = orig_step;
        } else if (g.pre && !g.gray) {   // the preprocessed frames are the magnifier's input
            a.dst_step = (size_t)g.dw * channels;
            CK(h->f_pre.grow(a.dst_step * g.dh * vl));
            a.dst = h->f_pre.p;
        }
        a.dst_lane_stride = a.dst_step * g.dh;
        if (g.gray) {
            CK(h->f_gray.grow((size_t)g.dw * g.dh * vl));
            a.gray = h->f_gray.p;
        }
        if (g.kind == FRONT_AREA && (st = area_tables(h, g, a)) != MC_OK) return st;
        if (std::any_of(h->hold.begin(), h->hold.end(), [](uint8_t x) { return x != 0; })) {
            h->f_flags_host.resize(vl);   // lives on the handle: the copy is asynchronous
            for (size_t v = 0; v < vl; ++v) h->f_flags_host[v] = !h->hold[v % lanes];
            CK(h->f_flags.grow(vl));
            CK(cudaMemcpyAsync(h->f_flags.p, h->f_flags_host.data(), vl, cudaMemcpyHostToDevice, h->stream));
            a.flags = h->f_flags.p;
        }
        const int src = nv ? FRONT_NV12 : channels == 3 ? FRONT_BGR : FRONT_GRAY;
        if ((st = launch_counted(h, "chain_front", [&] { return launch_chain_front(a, src, (int)vl, h->stream); })) != MC_OK) return st;
        mag_in = g.gray ? a.gray : a.dst;
        mag_step = g.gray ? (size_t)g.dw : a.dst_step;
    } else if (nv && p->mode != MC_MODE_NONE) {   // a plain NV12 -> BGR conversion
        if ((st = nv12_ingest(h, *nv, w, hh, (int)vl, p, false)) != MC_OK) return st;
        mag_in = h->n_in.p;
        mag_step = bgr_step_of(w);
    }

    // ---- the magnifier, straight into d_out; then the front's output for the frames it did not produce
    if ((st = clip_impl(h, mag_in, frames, g.dw, g.dh, g.cc, mag_step, p, d_out, out_step, produced)) != MC_OK) return st;
    info->magnified = std::any_of(produced, produced + vl, [](uint8_t x) { return x != 0; });
    if (!g.front()) return MC_OK;
    const size_t in_lane = mag_step * g.dh, out_lane = out_step * g.dh;
    return for_each_run(vl, [&](size_t v) { return !produced[v] && !h->hold[v % lanes]; }, [&](size_t a, size_t b) -> mc_status {
        CK(cudaMemcpy2DAsync(d_out + a * out_lane, out_step, mag_in + a * in_lane, mag_step, out_row, (b - a) * g.dh,
                             cudaMemcpyDeviceToDevice, h->stream));
        return MC_OK;
    });
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
    return chain_impl(h, d_in, in_step, nullptr, frames, width, height, channels, p, grayscale, d_out, out_step, d_original,
                      original_step, produced, info);
} catch (...) { return on_exception(h); }

extern "C" mc_status mc_chain_process_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                                  const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                                  uint8_t* d_original, size_t original_step, uint8_t* produced,
                                                  mc_chain_info* info) try {
    if (!h) return MC_ERR_INVALID;
    CK(cudaSetDevice(h->device));
    if (!in) { h->err = "NV12 plane is null"; return MC_ERR_INVALID; }
    return chain_impl(h, nullptr, 0, in, frames, width, height, 3, p, grayscale, d_out, out_step, d_original, original_step,
                      produced, info);
} catch (...) { return on_exception(h); }

// The one-lane host form: the frame is uploaded, runs the device chain, and what it wrote comes back tight.
extern "C" mc_status mc_chain_process(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                                      const mc_params* p, int grayscale, uint8_t* out, size_t out_bytes, uint8_t* original,
                                      size_t original_bytes, mc_chain_info* info) try {
    if (!h || !p || !info) return MC_ERR_INVALID;
    std::memset(info, 0, sizeof(*info));
    info->cur_is_input = 1; info->orig_is_input = 1;
    CK(cudaSetDevice(h->device));
    if (h->lanes != 1) { h->err = "mc_chain_process needs a 1-lane handle"; return MC_ERR_INVALID; }
    if (!h->inflight.empty()) { h->err = "mc_chain_process called with pipelined frames in flight"; return MC_ERR_INVALID; }
    if (h->hold[0]) { h->err = "mc_chain_process called while lane 0 is held"; return MC_ERR_INVALID; }
    const bool have = in != nullptr && width > 0 && height > 0;
    ChainGeom g;
    if (const char* e = chain_geometry(p, have ? width : 0, have ? height : 0, channels, grayscale, g, info)) {
        h->err = e;
        return MC_ERR_INVALID;
    }
    const size_t row = have ? (size_t)width * channels : 0, out_frame = (size_t)g.dw * g.dh * g.cc;
    const size_t orig_frame = (size_t)g.dw * g.dh * channels;
    if (have) {
        if (in_step < row) { h->err = "step too small"; return MC_ERR_INVALID; }
        CK(h->c_raw.grow(row * height));
        CK(h->c_out.grow(out_frame));
        if (g.pre) CK(h->c_orig.grow(orig_frame));
        CK(cudaMemcpy2DAsync(h->c_raw.p, row, in, in_step, row, (size_t)height, cudaMemcpyHostToDevice, h->stream));
    }
    uint8_t produced = 0;
    const mc_status st = chain_impl(h, have ? h->c_raw.p : nullptr, row, nullptr, 1, width, height, channels, p, grayscale, h->c_out.p,
                                    (size_t)g.dw * g.cc, g.pre ? h->c_orig.p : nullptr, (size_t)g.dw * channels, &produced, info);
    if (st != MC_OK || !have) return st;
    if (produced && info->cur_is_input) {   // no front stage: the magnified frame is the chain's result
        info->cur_is_input = 0; info->out_w = g.dw; info->out_h = g.dh; info->out_channels = g.cc;
    }
    if (!info->orig_is_input && original) {
        if (original_bytes < orig_frame) { h->err = "original buffer too small"; return MC_ERR_INVALID; }
        CK(cudaMemcpyAsync(original, h->c_orig.p, orig_frame, cudaMemcpyDeviceToHost, h->stream));
    }
    if (!info->cur_is_input && out) {
        if (out_bytes < out_frame) { h->err = "out buffer too small"; return MC_ERR_INVALID; }
        CK(cudaMemcpyAsync(out, h->c_out.p, out_frame, cudaMemcpyDeviceToHost, h->stream));
    }
    CK(cudaStreamSynchronize(h->stream));
    return MC_OK;
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
