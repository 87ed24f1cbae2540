// Per-mode device state + per-frame drivers: the H100 twins of magcore::MotionState / ColorState /
// RieszState and magnifyMotion / magnifyColor / magnifyRiesz (reference
// src/processing/magnification/MagnifyCore.hpp:24-40, :83-279).
#pragma once
#include <cufft.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/magcore_b200.h"
#include "mc_internal.h"

namespace mc {

// Optional per-launch event timing (bench roofline); events are drained by mc_profile_read.
struct Profiler {
    struct Rec { const char* name; int level; cudaEvent_t a, b; };
    std::vector<Rec> recs;
    bool begin(const char* name, int level, cudaStream_t s) {
        Rec r{name, level, nullptr, nullptr};
        if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return false;
        cudaEventRecord(r.a, s);
        recs.push_back(r);
        return true;
    }
    void end(cudaStream_t s) { cudaEventRecord(recs.back().b, s); }
};

// The handle's options (mc_set_option; each field is named as its key).
struct Options {
    bool faithful_level0 = false;
    bool keep_float_output = false;   // keep the pre-quantisation tap of the last frame (mc_get_float_output)
    bool profile_kernels = false;     // bracket every launch with events (mc_profile_read)
    bool use_tma = true;          // stage level-kernel tiles with cp.async.bulk.tensor
    bool egress_strip = true;     // Laplace egress as the register/shuffle strip kernel (false: the shared-memory tile kernel)
    bool band_from_state = true;  // synthesis rebuilds gain*(hi-lo) from the state planes instead of reading a stored band
                                  // (B200, with the state prefetch: level[1] 205 -> 177 us, egress +8 us)
    int lane_groups = 0;          // Laplace: number of lane groups run as concurrent launch chains (0 = automatic)
    bool analysis_only = false;   // Laplace / Phase: update the temporal state but skip synthesis + egress (*produced = 0); used
                                  // by the state-carry pass of temporal sharding (SURVEY 8f-3, lvm_b200.shard.magnify_segment)
    bool color_lane_lifecycle = false;   // a multi-lane Color handle accepts holds and single-lane restarts
};

struct ModeCtx {
    cudaStream_t stream;
    const DeviceTables* tables;
    uint64_t* launches;
    std::string* err;
    Options opt;       // the handle's, with one lane group while kernels are profiled
    float* float_out;  // optional [lanes][h][w][C] pre-quantisation tap
    Profiler* prof;    // optional
    // Lane lifecycle (mc_restart_lane / mc_hold_lane): the handle's LaneOp per lane for this frame, the device buffer the
    // mode uploads its per-lane ops to (stream-ordered: the previous frame's kernels have read it before the copy runs),
    // and the mode's answers: which lanes produced, and whether held lanes lost their state (reallocation, Phase cutoff change).
    const uint8_t* lane_ops = nullptr;   // host, `lanes` entries
    uint8_t* d_lane_ops = nullptr;       // device, `lanes` bytes
    uint8_t* lane_produced = nullptr;    // host, `lanes` entries, [t][lane] for a clip of t frames (written)
    bool* held_lost = nullptr;           // (written)
    // Per-lane parameters (mc_set_lane_params): each lane's effective parameters, `lanes` entries, when they are not all
    // the same; null when every lane runs with the call's (then the mode's `p` already carries them).
    const mc_params* lane_params = nullptr;
    uint8_t* lane_lost = nullptr;        // host, `lanes` entries (written): lanes whose state the mode dropped (a held one
                                         // restarts on release)
};

// The per-lane ops of one frame as a mode runs it: the handle's ops, with every lane that is not held turned into FIRST
// when the mode itself holds no state (first frame after allocation).
struct LanePlan {
    std::vector<uint8_t> op;
    int n_run = 0, n_first = 0, n_hold = 0;
    void make(const uint8_t* ops, int lanes, bool all_first) {
        op.assign(ops, ops + lanes);
        n_run = n_first = n_hold = 0;
        for (uint8_t& o : op) {
            if (all_first && o == LANE_RUN) o = LANE_FIRST;
            (o == LANE_HOLD ? n_hold : o == LANE_FIRST ? n_first : n_run)++;
        }
    }
    bool mixed() const { return n_hold > 0 || (n_run > 0 && n_first > 0); }
    // Mixed frames upload the ops and return the device array; uniform frames return null (the kernels' default path).
    cudaError_t upload(const ModeCtx& ctx, const uint8_t** d_ops) const {
        *d_ops = nullptr;
        if (!mixed()) return cudaSuccess;
        *d_ops = ctx.d_lane_ops;
        // pageable source: staged before the call returns, so `op` may change right after
        return cudaMemcpyAsync(ctx.d_lane_ops, op.data(), op.size(), cudaMemcpyHostToDevice, ctx.stream);
    }
    // The flags of `frames` frames ([t][lane]): frame 0 by each lane's op, every later frame `later_produces` for the
    // lanes that are not held (a clip's later frames run).
    void produced(const ModeCtx& ctx, bool run_produces, bool first_produces, int* any, int frames = 1,
                  bool later_produces = false) const {
        *any = 0;
        for (int t = 0; t < frames; ++t)
            for (size_t l = 0; l < op.size(); ++l) {
                const bool p = op[l] == LANE_HOLD ? false : t > 0 ? later_produces : op[l] == LANE_RUN ? run_produces : first_produces;
                ctx.lane_produced[(size_t)t * op.size() + l] = p ? 1 : 0;
                *any |= p ? 1 : 0;
            }
    }
};

// Launch bookkeeping shared by the mode drivers: counts the launch, optionally brackets it with events.
#define MCK(call)                                                             \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) {                                             \
            *ctx.err = std::string(#call) + ": " + cudaGetErrorString(e__);   \
            return MC_ERR_CUDA;                                               \
        }                                                                     \
    } while (0)
#define MCK_ST(call)                                                          \
    do {                                                                      \
        const mc_status s__ = (call);                                         \
        if (s__ != MC_OK) return s__;                                         \
    } while (0)
#define LAUNCH(name, level, call)                                             \
    do {                                                                      \
        const bool p__ = ctx.prof && ctx.prof->begin(name, level, ctx.stream);\
        cudaError_t e__ = (call);                                             \
        if (p__) ctx.prof->end(ctx.stream);                                   \
        if (e__ != cudaSuccess) {                                             \
            *ctx.err = std::string(name) + ": " + cudaGetErrorString(e__);    \
            return MC_ERR_CUDA;                                               \
        }                                                                     \
        ++*ctx.launches;                                                      \
    } while (0)

struct StateRef {  // a named state plane set for mc_get_state / mc_set_state
    float* ptr = nullptr;
    const int16_t* ptr16 = nullptr;   // read-only int16 planes ("lab16"), widened to f32 on download
    int rows = 0, cols = 0, channels = 0, pitch = 0;
    size_t plane_stride = 0;
    // floats from `ptr` to each lane's first plane, where the lanes are not channels * plane_stride apart (Color: the
    // pad float of odd lane blocks, and a ring slot of each lane's own); empty: lane * channels * plane_stride
    std::vector<size_t> lane_off;
    bool read_only = false;           // a tap of scratch the kernels overwrite every frame: mc_set_state refuses it
    bool found() const { return ptr || ptr16; }
};

// "lab16" (level 0, 3 channels): a mode's Lab16 planes of the last frame call, while they are current
inline void lab16_state(const int16_t* lab16, bool current, int w, int h, int pitch16, size_t plane16, StateRef& out) {
    out = StateRef{};
    if (!lab16 || !current) return;
    out.ptr16 = lab16; out.rows = h; out.cols = w; out.channels = 3; out.pitch = pitch16; out.plane_stride = plane16;
}

// One block of a lane's temporal state as mc_save_lane / mc_load_lane copy it: `rows` rows of `row_bytes` bytes,
// `pitch` bytes apart, from `ptr` (device).  A blob holds the rows dense.
struct LanePlane {
    void* ptr = nullptr;
    size_t pitch = 0, row_bytes = 0, rows = 0;
};

// Simple owner of cudaMalloc'ed float buffers (freed together on reset()).
struct DeviceArena {
    std::vector<void*> blocks;
    cudaError_t alloc(float** p, size_t floats);
    cudaError_t alloc_bytes(void** p, size_t bytes);
    void free_block(void* p);   // returns one block early (buffers replaced when a ring grows)
    void release();
};

// Scratch of a mode's clip path (mc_process_clip_device): the per-frame buffers of `cap` virtual lanes (frame t of lane k
// is virtual lane t * lanes + k).  The temporal state stays in the mode's own planes, so clip and frame calls interleave.
// A mode's Clip derives from this and adds its own planes and tensor maps.
struct ClipScratch {
    int cap = 0;                  // virtual lanes the buffers hold (the largest clip seen)
    int16_t* lab16 = nullptr;     // Lab planes of every frame (C == 3)
    float* fout = nullptr;        // pre-quantisation tap of every frame (keep_float_output)
    uint8_t* d_vops = nullptr;    // device LaneOp per virtual lane
    std::vector<uint8_t> vops;
    DeviceArena arena;

    // Grows `clip` to `vlanes` virtual lanes of `lane_floats` tap floats and `lab_bytes` Lab16 bytes (none when 0).  On
    // growth every buffer is released (cudaFree waits for the kernels still reading the old ones), `clip` starts over and
    // `alloc_planes()` allocates the mode's own planes.  The tap is added when keep_float_output first asks for it.
    template <class Clip, class AllocPlanes>
    static mc_status grow(Clip& clip, const ModeCtx& ctx, int vlanes, size_t lab_bytes, size_t lane_floats, AllocPlanes alloc_planes) {
        if (vlanes > clip.cap) {
            clip.arena.release();
            clip = Clip{};
            MCK_ST(alloc_planes());
            void* p = nullptr;
            if (lab_bytes) {
                MCK(clip.arena.alloc_bytes(&p, lab_bytes));
                clip.lab16 = (int16_t*)p;
            }
            MCK(clip.arena.alloc_bytes(&p, (size_t)vlanes));
            clip.d_vops = (uint8_t*)p;
            clip.cap = vlanes;
        }
        if (ctx.float_out && !clip.fout) MCK(clip.arena.alloc(&clip.fout, (size_t)clip.cap * lane_floats));
        return MC_OK;
    }
    // The ops of the clip's virtual lanes: HOLD for held lanes at every t, the plan's op at t = 0, RUN after.  With
    // `upload` they go to d_vops and *d_ops points there; otherwise *d_ops is null and every virtual lane runs.  Laplace
    // uploads for mixed plans only: a first frame is produced (its stored band is +-0), so when every lane takes one,
    // `first` alone describes the clip.  Phase uploads whenever a lane is not RUN: a first frame passes through, so the
    // kernels after the analysis must not write frame 0 of a FIRST lane, even when every lane is FIRST.
    cudaError_t upload_vops(const ModeCtx& ctx, const LanePlan& plan, int frames, bool upload, const uint8_t** d_ops);
    // The tap holds every frame of the clip: ctx.float_out gets the last frame of each lane that is not held, one copy
    // per run of such lanes.
    mc_status copy_last_tap(const ModeCtx& ctx, const LanePlan& plan, int frames, size_t lane_floats) const;
};

struct MotionMode {
    int lanes = 1;
    bool empty = true;       // MotionState::empty()
    bool allocated = false;
    int levels = 0, channels = 0, w = 0, h = 0;
    bool faithful = false;
    bool from_state = false;   // Options::band_from_state at allocation time
    std::vector<Level> lv;              // 0..levels
    std::vector<float*> G, hi, lo, M;   // per level (null where not kept)
    int16_t* lab16 = nullptr;           // Lab planes of the current frame (C == 3)
    int pitch16 = 0;
    size_t plane16 = 0;
    bool lab16_frame = false;           // lab16 holds the last frame call's Lab (clips write their own scratch)
    bool gauss_frame = false;           // G holds the last frame call's pyramid (clips write clip.G)
    // Every EMA step of the state since the state of all lanes was last dropped used cutoffs in [0, 1], so the a / b
    // state is bounded by the bands (a condition of L-only synthesis, DESIGN §4)
    bool ab_bounded = true;
    DeviceArena arena;

    // Lane groups (option "lane_groups"): the streams of a handle are independent, so their launch sets are issued as
    // `groups.size()` separate chains on separate CUDA streams.  A group's kernels no longer fill the GPU, so the block
    // scheduler co-schedules different stages of different groups on the same SMs — the L1-bound BGR->Lab ingest of one
    // group, the issue-bound egress of another and the HBM-bound level kernels of a third — instead of running the
    // stages back to back.  Buffers stay whole-handle allocations; a group sees them through offset pointers.
    struct Group {
        int lane0 = 0, lanes = 0;
        cudaStream_t stream = nullptr;     // null: the handle's stream (single group)
        cudaEvent_t done = nullptr;
        std::vector<TensorMapStorage> tmaps, tmaps_hi, tmaps_lo;   // per level: TMA descriptors of G[l] / hi[l] / lo[l] of this group's planes
        std::vector<char> tmap_valid;
    };
    std::vector<Group> groups;
    cudaEvent_t ev_fork = nullptr;
    int groups_req = 0;                    // Options::lane_groups at allocation time
    std::vector<float> gains;              // per-level gains of the current frame (member: no per-frame allocation)
    LanePlan plan;                         // per-lane ops of the current frame
    // The per-lane table of a frame whose lanes' parameters differ (ModeCtx::lane_params), on the device: per lane
    // {c_hi, 1 - c_hi, c_lo, 1 - c_lo}, per lane chroma, per level and lane the gain ([level][lane]).  Null members: every
    // lane uses the scalars.  coef_host is the device copy's contents.
    void* d_coef = nullptr;
    std::vector<uint8_t> coef_host;
    std::vector<double> coef_key;          // the lanes' six fields the table was built from (levels, w, h are the mode's)
    bool coef_in01 = true, coef_luma = true;   // the table's lanes' cutoff and L-only conditions
    const double* lane_ema = nullptr;
    const float *lane_chroma = nullptr, *lane_gain = nullptr;

    // Scratch of the clip path; the temporal state stays in hi / lo above.
    struct Clip : ClipScratch {
        std::vector<float*> G, M;             // per level: G_1 .. G_levels, amplified bands M_1 .. M_{levels-1}
        std::vector<TensorMapStorage> tmaps;  // per level: TMA descriptor of G_l over all virtual planes
        std::vector<char> tmap_valid;
    } clip;

    void reset();
    // frames > 1: `frames` consecutive frames of every lane ([t][lane] in io's lane stride); ctx.lane_produced then
    // holds frames * lanes flags
    mc_status process(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int levels, int* produced, int frames = 1);
    void find_state(const char* name, int level, StateRef& out);
    // the state of every lane for this key, as a frame call allocates it (every lane's next frame is its first)
    mc_status allocate(const ModeCtx& ctx, int w, int h, int channels, int levels);
    // lane `lane`'s state: hi then lo of every kept level, all channels of a plane set in one block
    void lane_planes(int lane, std::vector<LanePlane>& out) const;

private:
    mc_status make_groups(const ModeCtx& ctx);
    void drop_groups();
    bool luma_only(const ModeCtx& ctx) const;
    mc_status lane_table(const ModeCtx& ctx, bool* cutoffs_in_01, bool* luma_ok);
    const float* gain_of(int l, int lane0) const { return lane_gain ? lane_gain + (size_t)l * lanes + lane0 : nullptr; }
    mc_status run_group(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, Group& g, bool first, double c_lo, double c_hi,
                        bool luma);
    mc_status run_clip(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int frames, bool first, double c_lo, double c_hi,
                       bool luma);
    // the launch set around the level kernels, shared by run_group and run_clip
    bool fused_ingest() const;
    int first_level() const;
    mc_status ingest(const ModeCtx& ctx, const FrameIO& io, int16_t* lab, float* g1);
    LevelArgs level_args(int l, const std::vector<float*>& g, size_t p0, const int16_t* lab, const FrameIO& io, bool first,
                         double c_lo, double c_hi) const;
    mc_status copy_residual(const ModeCtx& ctx, const float* g_res, int lane0, int n);
    mc_status egress_first_frames(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, float* fout,
                                  bool first);
    mc_status egress(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, const BandSrc& m1,
                     const BandSrc& c2, float* fout, bool first_only, bool luma);
    template <class Band, class Out>
    mc_status synthesize(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, float* fout, bool motion,
                         bool luma, Band band, Out out);
};

// One lane's row of the Color kernels' per-lane table (uploaded on the handle's stream when the lanes are not uniform)
struct ColorLane {
    int src_head, src_mod, copy_n;   // relayout: destination slot t < copy_n <- source slot (src_head + t) % src_mod
    int append;                      // slot the frame is appended to; -1: held
    int n;                           // DFT length this frame; 0: the lane does not run the filter (does not produce)
    int sel;                         // physical slot of the reconstructed column (logical min(1, n - 1))
    float sc;                        // DFT scale of both transforms, 1 / n^2
    double fl, fh;                   // the CCS mask's packed index range for this n
    float amp;                       // the lane's amplification (read by k_select when lanes differ)
};

// A 2nd-order Butterworth section as the Phase kernels read it: numerator b0..b2, denominator a1, a2 (a0 = 1)
struct Butter { double b0, b1, b2, a1, a2; };
// One lane's row of the Phase kernels' per-lane table (uploaded when the lanes' designs or amplifications differ)
struct RieszLane {
    Butter lo, hi;                   // the lane's two filters
    float alpha, thresh;             // amplification and its clip (k_riesz_amplify)
    int rebuild_old;                 // the lane's cutoffs changed this frame: its prior is this frame's pyramid
};

struct ColorMode {
    int lanes = 1;
    bool allocated = false;
    int levels = 0, channels = 0, w = 0, h = 0;
    // Per lane: the rolling window's length, the physical slot of its OLDEST column and its logical ring size
    // max(getOptimalBufferSize(int(framerate)), length, 2).  head == 0 or count == mod, lane by lane.
    std::vector<int> count, head, mod;
    std::vector<ColorLane> table;   // host copy of this frame's per-lane table
    ColorLane* d_table = nullptr;
    std::vector<Level> lv;  // gaussian chain levels 0..levels
    std::vector<float*> G;  // pyrDown chain scratch (levels 1..levels-1) ; small level goes to the ring
    std::vector<float*> U;  // up-chain scratch
    std::vector<Level> ulv;
    float* ring = nullptr;      // [planes][rowsP][cap] time-major rows: each pixel's samples contiguous
    float* work = nullptr;      // gathered/filtered window [planes*rows][n]
    cufftComplex* spec = nullptr;
    float* minmax = nullptr;    // device scalars
    int small_rows = 0;         // pixels of the small level
    int ring_cap = 0;           // physical slots allocated (>= every lane's mod)
    struct FftPlans { cufftHandle r2c = 0, c2r = 0; size_t work_bytes = 0; void* bound = nullptr; };
    // per (DFT length, one lane): the window length (2 ... cap during warm-up) over all plan_signals signals, or over one
    // lane's channels * pixels signals (lanes whose windows differ in length)
    std::map<std::pair<int, bool>, FftPlans> plans;
    size_t plan_signals = 0;
    void* fft_work = nullptr;        // one work area shared by all cached plans (they run back to back on one stream)
    size_t fft_work_bytes = 0;
    DeviceArena arena;
    LanePlan plan;                   // per-lane ops of the current frame
    int tap_frame = -1;              // the taps' frame in the clip scratch (the last clip's last frame); -1: the frame planes
    std::vector<int> want_cap;       // per lane: the window cap its frame rate asks for (MagnifyCore.hpp:176)

    // What one frame's rows of the lane table ask of the filter
    struct Step {
        int n_filter = 0, n_max = 0;   // the first and the largest DFT length of a filtering lane (0: no lane filters)
        bool one_length = true;        // every filtering lane has the same length: one transform over all lanes
        bool uniform = true;           // every lane appends to the same slot and filters the same columns (scalar path)
    };

    // Scratch of the clip path: the per-frame planes of `cap` virtual lanes (frame t of lane k is virtual lane
    // t * lanes + k), one filtered window per frame, and the lane table of every virtual lane.  The window ring stays the
    // mode's own, so clip and frame calls interleave.
    struct Clip : ClipScratch {
        std::vector<float*> G, U;         // the Gaussian chain and the up chain (+ resized plane) of every virtual lane
        float* work = nullptr;            // frame t's filtered window at work + t * win_stride
        size_t work_floats = 0, win_stride = 0;
        unsigned* minmax = nullptr;       // per virtual lane: window min / max, then output min / max
        ColorLane* d_table = nullptr;
        std::vector<ColorLane> table;     // host rows, [t][lane]
        std::vector<Step> steps;          // per frame
    } clip;

    void reset();
    // frames > 1: `frames` consecutive frames of every lane ([t][lane] in io's lane stride); ctx.lane_produced then
    // holds frames * lanes flags
    mc_status process(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int levels, int* produced, int frames = 1);
    void find_state(const char* name, int level, StateRef& out);
    // the planes of this key with every window empty, as a frame call allocates them (the ring follows on the first frame)
    mc_status allocate(const ModeCtx& ctx, int w, int h, int channels, int levels);
    // lane `lane`'s window of `mod` slots as it lies in the ring: its block of physical slots 0 .. mod-1
    void lane_planes(int lane, int lane_mod, std::vector<LanePlane>& out) const;
    // makes the ring hold at least `need` slots, every lane's window in the slots it occupies (mc_load_lane)
    mc_status reserve_ring(const ModeCtx& ctx, int need);

private:
    // A slot's layout.  One lane's block of a slot is lane_sig() signals (pixels x channels).  cuFFT takes a lane's block
    // as the base pointer of a one-lane transform, which must be 8-byte aligned: on a multi-lane handle an odd block is
    // followed by one padding signal.
    size_t lane_sig() const { return (size_t)channels * small_rows; }
    size_t lane_stride() const { return lane_sig() + (lanes > 1 ? (lane_sig() & 1) : 0); }
    size_t slot_signals() const { return (size_t)lanes * lane_stride(); }
    // the ring grown to `need` slots (grow) or rotated; with `relayout` the lanes' windows move by d_rows' relayout fields
    mc_status reshape_ring(const ModeCtx& ctx, int need, bool grow, bool relayout, const ColorLane* d_rows);
    mc_status fft_plan(const ModeCtx& ctx, int n, bool one_lane, FftPlans** out);
    mc_status alloc_clip(const ModeCtx& ctx, int vlanes, size_t work_floats);
    // the append and filter rules of one frame: writes its `lanes` rows of a lane table, moves count / head
    // (lp: each lane's params, or null when every lane has p's; want_cap: each lane's window cap)
    Step step(const mc_params& p, const mc_params* lp, const std::vector<int>& want_cap, ColorLane* rows);
    // the launch sets shared by the frame and the clip path, over `vl` (virtual) lanes
    mc_status ingest(const ModeCtx& ctx, const FrameIO& io, int vl, const std::vector<float*>& g);
    mc_status filter(const ModeCtx& ctx, const Step& s, const ColorLane* rows, const ColorLane* d_rows, const float* top, float* win);
    mc_status reconstruct(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int vl, const ColorLane& row0, const ColorLane* tab,
                          const std::vector<float*>& g, const std::vector<float*>& u, const float* win, size_t win_stride,
                          unsigned* mm, int fout_v0);
};

struct RieszMode {
    int lanes = 1;
    bool allocated = false;     // st.cur != null
    int levels = 0, w = 0, h = 0;
    // Per lane: itsFrequency / itsFramerate of the two filters and their design.  The framerate is fixed when the lane's
    // design is made from scratch (the handle's state is built, or the lane's design was not finite), as the reference
    // fixes it at construction; a cutoff change re-designs at that framerate.
    struct Design {
        double lo_freq = 0, hi_freq = 0, framerate = 0;
        double loA[3] = {1, 0, 0}, loB[3] = {0, 0, 0}, hiA[3] = {1, 0, 0}, hiB[3] = {0, 0, 0};
        bool finite() const { return !std::isnan(loA[0]) && !std::isnan(hiA[0]); }
    };
    std::vector<Design> design;
    // lane k's next frame makes its design afresh at its params' framerate, as a structural reset of the handle would
    void redesign(int k) { if ((size_t)k < design.size()) design[(size_t)k].loA[0] = NAN; }
    std::vector<RieszLane> rows, rows_dev;   // this frame's per-lane table and the contents of its device copy
    RieszLane* d_rows = nullptr;
    std::vector<uint8_t> lane_ops;           // the handle's ops with lanes of a non-finite design turned FIRST
    std::vector<Level> lv;      // octave sizes, 0..levels-1 (band levels 0..levels-2 + low-pass residual)
    DeviceArena arena;
    // per level planes (one plane per lane: only L is processed)
    std::vector<float*> oct;                                  // octave i (input of level i); oct[levels-1] is the residual
    std::vector<float*> cur_low, cur_rx, cur_ry;              // this frame's band + Riesz pair
    std::vector<float*> old_low, old_rx, old_ry;              // prior pyramid (RieszState::old)
    std::vector<float*> phase_c, phase_s;                     // accumulated phase (the two filters' copies are identical)
    std::vector<float*> lo_r0c, lo_r0s, lo_r1c, lo_r1s, hi_r0c, hi_r0s, hi_r1c, hi_r1s;   // DF-II registers
    std::vector<float*> amp, t_c, t_s, low_amp, res;
    int16_t* lab16 = nullptr;
    int pitch16 = 0;
    size_t plane16 = 0;
    bool lab16_frame = false;   // lab16 holds the last frame call's Lab (clips write their own scratch)
    // How far the last frame call got, for the read-only taps (valid while lab16_frame): the octaves; + the phase kernel's
    // amp / t_c / t_s (some lane ran it); + the amplified band and the collapse (amplify ran)
    enum { TAPS_OCT = 1, TAPS_PHASE = 2, TAPS_SYNTH = 3 };
    int frame_taps = 0;
    // TMA descriptors of the 9x9 kernels' input tiles (72 x 24 boxes): octave i (analysis), amplified band i (collapse)
    std::vector<TensorMapStorage> tm_oct, tm_band;
    std::vector<char> tm_valid;
    LanePlan plan;              // per-lane ops of the current frame

    // Scratch of the clip path; the temporal state stays in the planes above.
    struct Clip : ClipScratch {
        std::vector<float*> oct;              // per level: octave i of every frame (oct[levels-1]: the residual)
        std::vector<float*> band, rx, ry;     // per band level: band and Riesz pair of every frame; after amplify, rx
                                              // holds the amplified band and band the collapse result
        float *amp = nullptr, *t_c = nullptr, *t_s = nullptr;   // one band level (the largest): phase_clip(i) and
                                                                // amplify(i) are issued back to back
        // per band level: TMA descriptors over all virtual planes of octave i (analysis), the band (phase_clip's
        // 40 x 20 window) and the amplified band (collapse)
        std::vector<TensorMapStorage> tm_oct, tm_band, tm_amp;
        std::vector<char> tm_valid;
    } clip;

    void reset();
    // frames > 1: `frames` consecutive frames of every lane ([t][lane] in io's lane stride); ctx.lane_produced then
    // holds frames * lanes flags
    mc_status process(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int levels, int* produced, int frames = 1);
    void find_state(const char* name, int level, StateRef& out);
    // The handle's state for `levels` levels at w x h, the filters designed from p (each lane's params) or, with p null,
    // not designed (not finite: the lane's next frame designs them, as a first frame)
    mc_status allocate(const ModeCtx& ctx, int w, int h, const mc_params* p, int levels);
    // lane `lane`'s state: the 13 planes of every band level, plane by plane (old.lowpass, old.rx, old.ry, phase.c,
    // phase.s, lo.r0.c, lo.r0.s, lo.r1.c, lo.r1.s, hi.r0.c, hi.r0.s, hi.r1.c, hi.r1.s)
    void lane_planes(int lane, std::vector<LanePlane>& out) const;

private:
    mc_status apply_cutoffs(const ModeCtx& ctx, const mc_params& p, std::vector<uint8_t>& rebuild);
    // the per-lane table of this frame (null when every lane's row is lane 0's: the scalars of row 0), uploaded on change
    mc_status lane_table(const ModeCtx& ctx, const mc_params& p, const std::vector<uint8_t>& rebuild, const RieszLane** d);
    mc_status frame_loop(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int levels, int* produced, int frames);
    mc_status run_clip(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int frames, bool first, int* produced);
    // the kernels shared by the frame and the clip path, over io.lanes lanes with io.ops
    mc_status build_pyramid(const ModeCtx& ctx, const FrameIO& io, int16_t* lab, const std::vector<float*>& octs,
                            const std::vector<float*>& bands, const std::vector<TensorMapStorage>& tm, const std::vector<char>& valid);
    mc_status amplify(const ModeCtx& ctx, const RieszLane* tab, int i, int n, const uint8_t* ops, const float* a, const float* tc,
                      const float* ts, const float* low, const float* rx, const float* ry, float* out);
    mc_status collapse_egress(const ModeCtx& ctx, const FrameIO& io, const int16_t* lab, const float* residual,
                              const std::vector<float*>& bands, const std::vector<float*>& out, const std::vector<TensorMapStorage>& tm,
                              const std::vector<char>& valid, float* fout);
};

}  // namespace mc
