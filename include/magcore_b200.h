/*
 * magcore_b200.h — C ABI of the H100-native Eulerian video-magnification core.
 *
 * Drop-in boundary: the reference's per-frame hot path sits behind
 *     livim::IProcessor::process(const FrameRef&, const ProcessorConfig&) / reset()
 *     (reference src/processing/IProcessor.hpp:50-60) as implemented by
 *     livim::MagnificationProcessor (src/processing/MagnificationProcessor.cpp:10-67).
 * One mc_handle == one MagnificationProcessor instance (it owns all temporal state, one CUDA
 * stream, no globals); `mc_process` has exactly that method's semantics on raw host pixels.
 *
 * Everything is extern "C", plain pointers and sizes; no exceptions cross this boundary (the C++
 * adapter in live-video-magnification_b200/adapter/ rethrows MC_ERR_* as std::runtime_error so the
 * reference's exception firewall, src/processing/ProcessingChain.cpp:50-62, keeps working).
 */
#ifndef MAGCORE_B200_H
#define MAGCORE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MC_ABI_VERSION 2

typedef struct mc_handle mc_handle;

typedef enum mc_status {
    MC_OK = 0,
    MC_ERR_INVALID = 1,     /* bad argument */
    MC_ERR_CUDA = 2,        /* a CUDA runtime / cuFFT call failed; see mc_last_error() */
    MC_ERR_NO_DEVICE = 3,   /* no usable sm_90 device: the core has no CPU fallback */
    MC_ERR_UNSUPPORTED = 4,
    MC_ERR_INTERNAL = 5     /* a C++ exception (std::bad_alloc, ...) was caught at the boundary; the handle's temporal
                               state has been dropped, as after any failed frame; see mc_last_error() */
} mc_status;

#define MC_MAX_LANES 4096   /* upper bound of mc_create_lanes(): lanes * channels is a CUDA grid.z extent */

/* livim::MagnificationMode, src/processing/IProcessor.hpp:10 (same numeric order). */
typedef enum mc_mode { MC_MODE_LAPLACE = 0, MC_MODE_PHASE = 1, MC_MODE_COLOR = 2, MC_MODE_NONE = 3 } mc_mode;

/* POD copy of livim::MagnificationParams (IProcessor.hpp:14-23) plus the PreprocessParams
 * fingerprint (IProcessor.hpp:26-41) which only takes part in the structural-reset decision
 * (src/processing/magnification/MagnifyCore.hpp:53-65).  Units are ALGORITHM units: Laplace
 * coLow/coHigh are EMA blend coefficients, Color/Phase cutoffs are Hz. */
typedef struct mc_params {
    int32_t mode;              /* mc_mode */
    int32_t levels;
    double amplification;
    double coWavelength;
    double coLow;
    double coHigh;
    double chromAttenuation;
    double framerate;
    int32_t pre_downscale;     /* PreprocessParams::downscale */
    int32_t pre_roiEnabled;
    float pre_roiX, pre_roiY, pre_roiW, pre_roiH;
} mc_params;

/* Fills *p with the reference defaults (MagnificationParams{} + PreprocessParams{}). */
void mc_params_default(mc_params* p);

/* UI units -> algorithm units; replaces livim::toParams(), src/processing/MagnificationParamsUi.hpp:74-103
 * (amplification, wavelength %, low/high Hz, chroma %, levels, captureFps). */
void mc_params_from_ui(mc_params* p, int mode, int amplification, double wavelength, double low_hz,
                       double high_hz, int chroma, int levels, double fps);

/* livim::calculateMaxLevels, src/processing/magnification/SpatialFilter.cpp:5-11. */
int mc_calculate_max_levels(int width, int height);

/* livim::getOptimalBufferSize, src/processing/magnification/TemporalFilter.cpp:82-94. */
int mc_optimal_buffer_size(int fps);

/* livim::butterworth(N, Wn, a, b), src/processing/magnification/TemporalFilter.cpp:279-297;
 * a and b must hold N+1 doubles. */
mc_status mc_butterworth(unsigned order, double wn, double* a, double* b);

/* Per-level Laplace gains, src/processing/magnification/MagnifyCore.hpp:114-134; gains[levels+1]. */
mc_status mc_motion_gains(const mc_params* p, int levels, int width, int height, float* gains);

int mc_abi_version(void);
int mc_device_count(void);

/* Construct / destroy a processor bound to CUDA device `device` (replaces
 * std::make_unique<MagnificationProcessor>(), src/processing/ChainBuilder.cpp:15).
 * `lanes` >= 1 independent streams are stepped in lock-step by one handle (lanes == 1 is the
 * reference's processor; lanes > 1 is the throughput form: one launch set serves all lanes,
 * each lane keeping its own temporal state — used for multi-stream serving and for benchmarking
 * against a working set larger than L2; mc_restart_lane / mc_hold_lane give each lane its own lifecycle). */
mc_status mc_create(int device, mc_handle** out);
mc_status mc_create_lanes(int device, int lanes, mc_handle** out);
void mc_destroy(mc_handle* h);

/* MagnificationProcessor::reset(), MagnificationProcessor.cpp:10-15.  Every lane's next frame is its first frame;
 * holds (mc_hold_lane) are kept. */
mc_status mc_reset(mc_handle* h);

/* --- lane lifecycle: each lane of a multi-lane handle behaves like its own MagnificationProcessor -------------------
 * A frame call computes one op per lane: HOLD if the lane is held; otherwise FIRST if the lane has no temporal state
 * (after mc_create_lanes, mc_reset, mc_restart_lane, a structural change — size, levels, channels, mode, preprocess —
 * mode None or a failed frame); otherwise RUN.  Restarts and holds are taken when a frame is submitted or processed;
 * frames already in flight are not affected.  Per mode:
 *   Laplace: FIRST is the reference's first frame for that lane (MagnifyCore.hpp:98-103): hi = lo = band, the output is
 *            the input round-tripped through Lab, and it is produced.
 *   Phase:   FIRST passes the lane through (not produced) and makes this frame its `old` pyramid with a zero Riesz pair and
 *            zeroed phases / filter registers (MagnifyCore.hpp:226-240).  A cutoff change while a lane is held drops that
 *            lane's state: its first frame after release is FIRST.
 *   Color:   each lane has its own rolling window.  FIRST restarts it empty and appends the frame: one column, not
 *            produced (MagnifyCore.hpp:180).  RUN appends; the lane produces from two columns on.  HOLD leaves the
 *            window as it is.  A frame-rate change applies to each lane's own window when the lane next runs.  With
 *            option "color_lane_lifecycle" = 1 every lane then equals, bit for bit, its own 1-lane handle fed its
 *            frames.  Without it (the default) a frame call on a handle with lanes > 1 while a lane is held, or while
 *            some lanes are restarted and others run, returns MC_ERR_UNSUPPORTED and changes nothing.  With lanes == 1
 *            a held handle skips frame calls entirely (the window is unchanged). */

/* The lane's next frame is its first frame: the lane's temporal state is dropped, the other lanes are untouched.
 * On a 1-lane handle this is mc_reset().  MC_ERR_INVALID if lane is out of range. */
mc_status mc_restart_lane(mc_handle* h, int lane);

/* hold != 0: until released, frame calls skip this lane.  Its temporal state is left exactly as it is, its bytes of
 * `out` are not written, and its produced flag is 0.  Holds are sticky and survive mc_reset and structural resets
 * (a structural reset still drops the held lane's state: it restarts on release).  MC_ERR_INVALID if lane is out of
 * range.  mc_chain_process returns MC_ERR_INVALID while lane 0 is held. */
mc_status mc_hold_lane(mc_handle* h, int lane, int hold);

/* --- per-lane parameters: each lane of a multi-lane handle with its own magnification parameters -------------------- */
/* The non-structural fields of mc_params, in the same (algorithm) units. */
typedef struct mc_lane_params {
    double amplification, coWavelength, coLow, coHigh, chromAttenuation, framerate;
} mc_lane_params;
/* lp != NULL: from the next frame call or submit on, `lane` uses these six fields in place of those of the call's
 * params; mode, levels and preprocess still come from the call.  lp == NULL: the lane follows the call's params again.
 * Effective params "differ" when their fields differ bit for bit (+0 / -0 can step the state into different bits).
 *   Equivalence: lane k's effective params at a frame are the call's mc_params with the six fields replaced by lane k's
 *     override, if it has one.  Lane k then gives, bit for bit, what a 1-lane handle gives when fed lane k's frames with
 *     those params, under the restarts and holds it saw: the output bytes, the produced flag, mc_lane_produced and the
 *     temporal state afterwards.
 *   Where it applies: every call that runs the magnifier — frame calls, clips (the override is taken at the clip's first
 *     frame, like restarts and holds), chain, compose, NV12 and YUYV / UYVY calls, and every submit.  For pipelined
 *     submits the override is taken at submit: frames already in flight keep the params they were submitted with.
 *   Lifetime: an override is configuration, not temporal state.  It survives mc_reset, structural resets and failed
 *     frames, as holds and the overlay do, until it is replaced or cleared.
 *   Laplace: each lane's gains, EMA coefficients and chroma attenuation come from its own params.
 *   Phase: each lane keeps its own filter design (itsFrequency / itsFramerate), with the framerate fixed when the lane's
 *     design is made from scratch: when the handle's state is built (every lane's first frame at once, as after
 *     mc_reset) or when the lane's design was not finite.  A cutoff change on one lane re-designs only that lane's
 *     filters at its framerate, zeroes only its registers and rebuilds only its `old`; a held lane whose cutoffs change
 *     drops its state and restarts on release.  A lane restarted alone (mc_restart_lane) keeps its design's framerate:
 *     after a framerate change its 1-lane twin, restarted with mc_reset, re-designs at the new rate, so the two differ
 *     from there on; this is the behaviour lanes without an override have always had.  A clip with a NaN cutoff runs as
 *     frame calls.
 *   Color: each lane's window cap comes from its own framerate, and its mask and amplification from its own params.  A
 *     Color handle with lanes > 1 whose lanes' effective params differ needs option "color_lane_lifecycle"; without it
 *     the frame call returns MC_ERR_UNSUPPORTED and changes nothing.
 * MC_ERR_INVALID for a NULL handle or a lane out of range. */
mc_status mc_set_lane_params(mc_handle* h, int lane, const mc_lane_params* lp);

/* --- per-lane region of interest: each camera of a multi-lane handle cropped at its own rectangle --------------------- */
/* roi != NULL: from the next frame call or submit on, `lane` uses the four floats roi[0..3] = {x, y, w, h} (normalised, as
 * pre_roiX / Y / W / H) in place of the call's ROI fields; pre_roiEnabled, pre_downscale, grayscale, mode and levels still
 * come from the call.  roi == NULL: the lane follows the call's ROI again.
 *   Equivalence: lane k's effective params are the call's, with the four ROI fields replaced by lane k's override if it has
 *     one.  Lane k then gives, bit for bit, what a 1-lane handle gives when fed lane k's frames with those params, under
 *     the restarts and holds lane k saw: the processed frame and the original tap, the canvas (labels included), `info`,
 *     the produced flags, mc_lane_produced, and the temporal state afterwards (which a mc_save_lane blob shows byte for
 *     byte).
 *   Where it applies: every call.  Chain, compose, clip and submit calls of every source (BGR, gray, NV12, 4:2:2, I420,
 *     RGB) crop each lane's frames at the lane's own rectangle.  The magnifier-only calls (mc_process*, mc_submit*) do not
 *     crop, so there the override only enters the lane's structural fingerprint.  A clip takes the override at its first
 *     frame and a submit at submit time: frames in flight keep what they were submitted with.
 *   Per-lane structural reset: the fingerprint (mode, levels, size, channels, downscale, pre_roiEnabled and the ROI,
 *     compared with exact ==) is kept per lane.  A lane whose effective ROI changes while the rest stays restarts alone,
 *     as its 1-lane twin would; the other lanes continue untouched.  A Phase lane restarted this way re-designs its
 *     filters at its effective framerate, as its twin's structural reset does (mc_restart_lane keeps the design's
 *     framerate, see mc_set_lane_params).  A held lane keeps its state while its ROI changes: it is compared when the
 *     lane is released, which restarts it only if its ROI then differs from the one it ran with.  A change of the
 *     rest of the fingerprint, or of every lane's ROI at once, still resets every lane.  On a Color handle with lanes > 1,
 *     restarting some lanes needs option "color_lane_lifecycle": without it the call returns MC_ERR_UNSUPPORTED and
 *     changes nothing.
 *   One geometry: in a call that crops (pre_roiEnabled), every lane that runs must get a crop of the same pixel size after
 *     the rounding (lround) and clamping of PreprocessParams; that size is the call's output geometry.  Otherwise the call
 *     returns MC_ERR_INVALID before any copy or launch, with nothing changed, and mc_last_error names the lane.  Held lanes
 *     are checked when they run again.
 *   Lifetime: an override is configuration.  Like mc_set_lane_params and holds, it survives mc_reset, structural resets
 *     and failed frames.
 *   Lane state: a mc_save_lane blob records the saving lane's own fingerprint, ROI included.  A load into a handle that
 *     holds state must match the destination lane's own fingerprint (MC_ERR_INVALID otherwise); a load into a handle
 *     without state takes the blob's.  A later call whose effective ROI for that lane differs restarts the lane, as the
 *     source lane's twin would.
 * MC_ERR_INVALID for a NULL handle or a lane out of range. */
mc_status mc_set_lane_roi(mc_handle* h, int lane, const float* roi);

/* --- lane state: save one lane's temporal state as host bytes, and load it into a lane of any handle ------------------
 * A running stream moves (to another lane, handle, GPU, process or a file) without the visible restart of its temporal
 * filters: save its lane on the source, load the blob into the destination lane, then restart or hold the source lane.
 *   Equivalence: lane k of handle A is saved after some call, and the blob is loaded into lane j of handle B (any lane
 *     count, the same or another device, or A itself).  Fed lane k's next frames with the same effective parameters,
 *     through any mix of frame, clip, chain, compose, NV12, 4:2:2 and submit calls, lane j then gives, bit for bit, what
 *     lane k would have given: the output bytes, the produced flags, mc_lane_produced and the temporal state afterwards.
 *     B's other lanes equal, bit for bit, those of a twin of B without the load, and A those of a twin of A without the
 *     save: a save only reads.
 *   What travels: temporal state only.  The lane's "has state" bit: a lane without state saves a valid blob (without
 *     planes), and loading it is mc_restart_lane.  Laplace: hi / lo of every kept level (levels 0 and `levels` too with
 *     faithful_level0), and whether the state is bounded (a loaded unbounded state turns L-only synthesis off for B,
 *     DESIGN.md §4).  Phase: the 13 planes of every band level (those mc_get_state names) and the lane's filter design:
 *     its cutoffs, the framerate it was designed at and its coefficients, so a lane designed at 25 fps keeps that design
 *     in a handle whose other lanes run at 30 fps.  Color: the window's length, the physical slot of its oldest column,
 *     its ring size and its slots as they lie (not rotated into logical order: the filter's rounding follows the slots).
 *   What stays: configuration belongs to the destination lane: its hold, its mc_set_lane_params override and the handle's
 *     overlay and options.  Move an override yourself.  The read-only taps ("gauss", "lab16", "oct", "window", ...)
 *     describe the last frame call and are not changed by a load.  A held lane stays held and runs from the loaded state
 *     when it is released.
 *   Key: the blob records the structural key (mode, clamped levels, width, height, channels, the preprocess fingerprint)
 *     and, for Laplace, faithful_level0.  If B holds state (after a frame call of some mode), the blob's key must be its
 *     key; if it holds none (new, after mc_reset, a structural reset, mode None or a failed frame), the load takes the
 *     blob's key and allocates the mode's state as a frame call with that key would: every other lane has no state.  A
 *     later frame call with another key resets structurally, as always.
 *   Blocking: a save waits for the work enqueued on the handle, and a load has finished when it returns (src may be freed).
 *     Pageable buffers go through the handle's pinned staging (grow-only: the largest blob's planes); pinned ones are
 *     copied directly.
 *   Blob: opaque, stable within a blob version: a header (magic, version, total size, key, the mode's scalars), then the
 *     planes as dense rows.  Saving right after a load gives the same bytes.  1080p colour: Laplace at 6 levels 16.6 MB,
 *     Phase at 6 levels 143.6 MB, Color at 3 levels with a 64-slot window 24.9 MB.
 *   Errors, with no state, flag or configuration changed: MC_ERR_INVALID for a NULL handle, `bytes` or src; a lane out of
 *     range; cap smaller than the blob; a blob that is truncated (`bytes` is not its size) or of another magic or version;
 *     a key or faithful_level0 that differs from B's; submitted frames in flight.  MC_ERR_UNSUPPORTED for a load into a
 *     Color handle (or of a Color blob) with lanes > 1 without option "color_lane_lifecycle".  A CUDA failure while the
 *     planes are copied in drops B's state, as a failed frame does. */
/* Save lane `lane`'s temporal state into dst (host memory, pinned or pageable).  dst == NULL: only *bytes is set, to
 * the size needed.  Otherwise cap must be >= that size; *bytes receives the bytes written. */
mc_status mc_save_lane(mc_handle* h, int lane, void* dst, size_t cap, size_t* bytes);
/* Make lane `lane`'s temporal state the one saved in src (host memory, `bytes` long).  The other lanes are untouched. */
mc_status mc_load_lane(mc_handle* h, int lane, const void* src, size_t bytes);

/* Per-lane produced flags (n == lanes) of the frame most recently returned by mc_process / mc_process_device /
 * mc_chain_process, or collected by mc_collect.  The `*produced` of those calls is "at least one lane produced", and
 * a lane's bytes of `out` are written only when its flag is 1.  MC_ERR_INVALID if n != lanes. */
mc_status mc_lane_produced(mc_handle* h, uint8_t* produced, int n);

/* MagnificationProcessor::process(), MagnificationProcessor.cpp:17-67, on host pixels.
 *   in   : `lanes` frames back to back, each h rows of `in_step` bytes, CV_8UC3 BGR interleaved
 *          (channels == 3) or CV_8UC1 (channels == 1); treated as immutable.
 *   out  : same geometry with `out_step`; lane i's frame is written only when lane i produced (mc_lane_produced).
 *   *produced == 0  <=>  no lane produced: the reference returns the input FrameRef unchanged (mode None, empty or
 *          too-small image, Color warm-up, Riesz first frame / gray input, held lanes).
 * Blocking: H2D copy, kernels and D2H copy complete before it returns. */
mc_status mc_process(mc_handle* h, const uint8_t* in, int width, int height, int channels,
                     size_t in_step, const mc_params* p, uint8_t* out, size_t out_step,
                     int* produced);

/* Same contract on DEVICE pointers (frames already resident in HBM; lane stride = h*step).
 * Work is enqueued on the handle's stream; call mc_sync() before reading d_out on another stream. */
mc_status mc_process_device(mc_handle* h, const uint8_t* d_in, int width, int height, int channels,
                            size_t in_step, const mc_params* p, uint8_t* d_out, size_t out_step,
                            int* produced);
mc_status mc_sync(mc_handle* h);

/* --- clips: T = `frames` consecutive frames of every lane in one call (an exporter that knows its clip up front) -----
 * in/out hold frame t of lane k at (t * lanes + k) * height * step.  produced: frames * lanes bytes, [t][lane].  The
 * result (out bytes, produced flags, temporal state afterwards, mc_lane_produced = the last frame's flags) is exactly
 * that of `frames` consecutive mc_process_device calls with the same params and no lifecycle calls in between:
 * restarts and holds are taken at the clip's first frame, and a held lane is skipped for the whole clip.  A frame that
 * did not produce leaves its bytes of out untouched.
 *   Laplace: one launch set for the whole clip.  The spatial kernels run over frames * lanes "virtual lanes", and the
 *            level kernel carries each tile's temporal state in registers from the first frame to the last, so the
 *            state planes are read and written once per clip instead of once per frame.  The structural tracker runs
 *            once, at the clip's first frame; analysis_only produces only the lanes' first frames, as frame calls do.
 *   Phase:   one launch set for the whole clip as well.  The analysis, amplification, collapse and egress run over
 *            the virtual lanes, and the phase kernel carries each pixel's prior pyramid, phases and Butterworth
 *            registers in registers across the clip.  A filter design that is not finite (every frame is a first frame)
 *            runs as frame calls.  analysis_only updates the state and produces nothing, as frame calls do.
 *   Color:   one launch set for the whole clip, apart from the window filter.  The ingest, the Gaussian chain and
 *            everything after the filter (window min / max, column select, pyrUp chain, resize, output stretch) run
 *            over the virtual lanes; the append to the window and its DFT pair run frame by frame, as in frame calls.
 *            The read-only taps ("gauss", "window", "filtered", "up") after a clip are those of its last frame.
 * MC_ERR_INVALID, with the state untouched, when frames < 1, frames * lanes > MC_MAX_LANES, produced is NULL or frames of
 * mc_submit are in flight; the parameter checks of mc_process_device apply unchanged.  Mode None and an empty image
 * are the identity (all flags 0, state dropped).  A failed clip drops the state like a failed frame.  The clip path
 * keeps device scratch for the largest clip seen, released by mc_reset: ~29 MB (Laplace) or ~82 MB (Phase) per 1080p
 * colour frame at 6 levels, ~91 MB (Color, 64-frame window, 3 or 6 levels). */
mc_status mc_process_clip_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                 size_t in_step, const mc_params* p, uint8_t* d_out, size_t out_step, uint8_t* produced);
/* The same on host pointers, blocking (upload, kernels, download of the produced frames only).  Pinned or pageable. */
mc_status mc_process_clip(mc_handle* h, const uint8_t* in, int frames, int width, int height, int channels,
                          size_t in_step, const mc_params* p, uint8_t* out, size_t out_step, uint8_t* produced);

/* --- the whole processing chain on the device (SURVEY.md 8f-1) -----------------------------------------------------
 * Replaces runChainOnce(chain, in, cfg, original) (reference src/processing/ChainBuilder.cpp:19-29) over
 * PreprocessProcessor (ROI crop + INTER_AREA downscale, PreprocessProcessor.cpp:10-51), GrayscaleProcessor
 * (BGR2GRAY, GrayscaleProcessor.cpp:7-16) and MagnificationProcessor: both front stages run bit-exact on the H100 in
 * one kernel ("chain_front" in profile_kernels), the magnification core runs on their result, and the processed frame
 * plus the "original" tap (the pre-magnification frame, ChainBuilder.cpp:25) are written.
 * mc_chain_process: one host frame, lanes must be 1, blocking; MC_ERR_INVALID while lane 0 is held.  `out` /
 * `original` are written tight (step = width * channels); the *_is_input flags mirror the reference returning the very
 * same FrameRef (nothing written). */
typedef struct mc_chain_info {
    int32_t cur_is_input;                    /* processed frame == the input FrameRef */
    int32_t out_w, out_h, out_channels;      /* geometry of `out` when cur_is_input == 0 */
    int32_t orig_is_input;                   /* original tap == the input FrameRef */
    int32_t orig_w, orig_h, orig_channels;   /* geometry of `original` when orig_is_input == 0 */
    int32_t magnified;                       /* the magnification stage produced a frame */
} mc_chain_info;
mc_status mc_chain_process(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                           const mc_params* p, int grayscale, uint8_t* out, size_t out_bytes, uint8_t* original,
                           size_t original_bytes, mc_chain_info* info);

/* The geometry runChainOnce gives a width x height x channels frame under p / grayscale, without a handle or a GPU:
 * info as mc_chain_process reports it for a frame the magnifier does not produce.  An empty frame (width or height
 * <= 0) is the identity.  MC_ERR_INVALID when p or info is NULL or channels is not 1 or 3. */
mc_status mc_chain_geometry(const mc_params* p, int width, int height, int channels, int grayscale, mc_chain_info* info);

/* runChainOnce for every lane and `frames` consecutive frames, on device frames, enqueued on mc_stream().
 *   Layout: virtual lane v = t * lanes + k is frame t of lane k.  It sits at v * height * in_step in d_in, at
 *     v * out_h * out_step in d_out and at v * orig_h * original_step in d_original (out_h / orig_h of `info`, or height
 *     where the stage is an identity).  produced: frames * lanes bytes, [t][lane].  frames == 1 is a frame call; frames
 *     > 1 follows the clip rules of mc_process_clip_device unchanged (lifecycle taken at the first frame, every mode
 *     batched, Color's window filter frame by frame).
 *   Equivalence: every virtual lane gets, bit for bit, what mc_chain_process on a 1-lane handle gives when fed that
 *     lane's frames in order: the processed frame, the original tap, the info and the temporal state afterwards (held
 *     lanes and Color's lanes as in the lane lifecycle above).
 *   What is written: `info` is mc_chain_geometry's, except that `magnified` is "at least one frame produced".  Virtual
 *     lane v's processed frame is written to d_out when produced[v] is set or when info.cur_is_input == 0 (a front
 *     stage ran); otherwise the input is the result, as the reference returns the same FrameRef.  d_original is written
 *     for every virtual lane that is not held when info.orig_is_input == 0 and d_original is not NULL.  Held lanes leave
 *     both buffers untouched.  mc_lane_produced reports the last frame's flags.
 *   Errors, returned before any kernel runs and with no caller buffer or state changed: MC_ERR_INVALID for steps smaller
 *     than a row, a NULL d_out when the call would write to it (a front stage is on or the mode is not None), frames < 1,
 *     frames * lanes > MC_MAX_LANES, NULL produced / info / params, or pipelined frames in flight; MC_ERR_UNSUPPORTED
 *     for Color's multi-lane refusals (without option "color_lane_lifecycle").  Mode None and an empty image are the
 *     identity for the magnifier: the front stages still run when they are on.
 *   Device scratch: the front keeps staging for its output (the preprocessed frames when d_original is NULL, the gray
 *   frames) and the INTER_AREA tap tables, which are uploaded on mc_stream() only when the crop or output size changes. */
mc_status mc_chain_process_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                  size_t in_step, const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                  uint8_t* d_original, size_t original_step, uint8_t* produced, mc_chain_info* info);

/* Pipelined host path: mc_submit enqueues H2D + kernels + D2H for one frame asynchronously on
 * three streams (copy-in, compute, copy-out) and returns; mc_collect waits for the OLDEST
 * outstanding frame (strict FIFO — frame order is preserved, as ProcessingChain.hpp:18-20 needs)
 * and reports whether `out` of that submit was written.  `in`/`out` that are pinned host memory
 * (cudaHostAlloc / cudaHostRegister / mc_host_alloc) are copied straight to/from HBM; pageable
 * buffers go through the handle's pinned staging slots.  At most mc_pipeline_depth() frames may
 * be in flight; `in` and `out` must stay valid until the frame is collected. */
int mc_pipeline_depth(mc_handle* h);
mc_status mc_submit(mc_handle* h, const uint8_t* in, int width, int height, int channels,
                    size_t in_step, const mc_params* p, uint8_t* out, size_t out_step);
mc_status mc_collect(mc_handle* h, int* produced);

/* The processing chain on host frames, pipelined: mc_chain_process_device with frames == 1 on host memory, submitted
 * and collected as mc_submit is.  One call submits one frame of every lane; mc_collect collects it, in strict FIFO
 * order with mc_submit, mc_submit_nv12 and the other chain submits on the handle.  `*produced` of mc_collect is "at
 * least one lane magnified", and mc_lane_produced then gives the lanes' flags (a chain submit does not change what
 * mc_lane_produced reports before its frame is collected).
 *   Layout: lane k of `in` at k * height * in_step (BGR or gray; NV12 and 4:2:2 frames: at k * lane_stride); lane k of
 *     `out` at k * out_h * out_step and of `original` at k * orig_h * original_step (out_h / orig_h of `info`, or height
 *     where the stage is an identity).  Each buffer may be pinned or pageable, independently of the others, and must stay
 *     valid until its frame is collected.
 *   What is written: that of mc_chain_process_device.  For each lane that is not held, `out` when the lane's flag is 1
 *     or info.cur_is_input == 0, and `original` when info.orig_is_input == 0 and original is not NULL.  Held lanes, row
 *     padding and the other lanes' bytes stay untouched.  For any sequence of submits and lifecycle, parameter or
 *     structural changes, the bytes written, the flags, mc_lane_produced and the temporal state equal, bit for bit, those
 *     of mc_chain_process_device (or its _nv12 / _yuv422 form) on the same frames uploaded by the caller; restarts,
 *     holds and parameters are taken at submit.
 *   info: filled by the submit, final when it returns; mc_chain_geometry's (for a 4:2:2 source both frames are written),
 *     with magnified 0: the collected *produced carries that fact.
 *   Errors, returned before any copy or kernel is enqueued, with the handle's state and the frames in flight unchanged:
 *     MC_ERR_INVALID for a full pipeline, slot buffers that would have to grow while frames are in flight ("pipeline
 *     geometry changed"), and every argument error of the matching device chain call (a NULL `out` where the call would
 *     write it included); MC_ERR_UNSUPPORTED for Color's multi-lane refusals.  A chain submit takes one frame
 *     per lane; clips are submitted through the compose submits (mc_chain_compose_submit, after the 4:2:2 section).
 * mc_chain_submit_nv12 and mc_chain_submit_yuv422 follow the NV12 and 4:2:2 sections below. */
mc_status mc_chain_submit(mc_handle* h, const uint8_t* in, int width, int height, int channels, size_t in_step,
                          const mc_params* p, int grayscale, uint8_t* out, size_t out_step, uint8_t* original,
                          size_t original_step, mc_chain_info* info);

/* --- NV12 frames: the hand-off format of hardware video decoders and encoders ---------------------------------------
 * NV12 is 4:2:0 YCbCr in two planes: a luma plane (height rows of width bytes) and a plane of interleaved Cb,Cr pairs
 * (height/2 rows of width bytes), one pair per 2x2 pixel block.  The matrix is ITU-R BT.601, limited range (Y 16..235,
 * Cb/Cr 16..240); chroma is sited at the top-left pixel of each block.  The core converts on the device exactly as
 * OpenCV does (u8, 20-bit fixed point): the input with cvtColor(COLOR_YUV2BGR_NV12), which gives every pixel of a block
 * the block's Cb,Cr; the output with cvtColor(COLOR_BGR2YUV_I420), whose Cb,Cr are those of each block's top-left pixel,
 * stored interleaved.  The magnifier in between sees 3-channel BGR frames, so for any NV12 input X an NV12 call gives
 *     out = to_nv12(bgr_call(to_bgr(X)))
 * bit for bit: the output bytes, the produced flags and the temporal state afterwards.  NV12 and BGR calls of the same
 * geometry interleave on one handle without a structural reset (the tracker sees channels = 3).  A lane or frame that
 * did not produce leaves both of its planes of `out` untouched.  keep_float_output, profile_kernels ("nv12_to_bgr",
 * "bgr_to_nv12"), the lane lifecycle and the clip rules apply unchanged.  MC_ERR_INVALID, with the state untouched, when
 * width or height is odd or < 2, pitch < width, a plane pointer is NULL, or (more than one lane) lane_stride is less
 * than pitch * height.  Each call keeps device BGR staging for the largest frame set seen. */
typedef struct mc_nv12 {
    uint8_t* y;          /* luma plane of lane 0 (of frame 0 of lane 0 in a clip): height rows of width bytes */
    uint8_t* uv;         /* interleaved Cb,Cr plane of the same frame: height/2 rows of width bytes; it need not follow
                            the luma plane (decoders put it at pitch * aligned height, e.g. 1088 rows for 1080p H.264) */
    size_t pitch;        /* bytes per row, both planes */
    size_t lane_stride;  /* bytes from one (virtual) lane's planes to the next, the same for y and uv */
} mc_nv12;
/* mc_process_device on NV12 device planes. */
mc_status mc_process_nv12_device(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p,
                                 const mc_nv12* out, int* produced);
/* mc_process_clip_device on NV12 device planes: frame t of lane k is virtual lane t * lanes + k of in / out;
 * produced: frames * lanes bytes, [t][lane]. */
mc_status mc_process_clip_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                      const mc_params* p, const mc_nv12* out, uint8_t* produced);
/* mc_submit on NV12 host planes, pinned or pageable; collected by mc_collect.  Only NV12 bytes cross PCIe (1.5 B/px
 * each way); pageable planes go through NV12-sized pinned staging.  There is no blocking host NV12 call: submit and
 * collect. */
mc_status mc_submit_nv12(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p, const mc_nv12* out);
/* mc_chain_submit on NV12 host planes (the checks of mc_chain_process_nv12_device): 1.5 B/px cross PCIe upwards. */
mc_status mc_chain_submit_nv12(mc_handle* h, const mc_nv12* in, int width, int height, const mc_params* p, int grayscale,
                               uint8_t* out, size_t out_step, uint8_t* original, size_t original_step, mc_chain_info* info);
/* mc_chain_process_device on NV12 device planes: see the chain section above. */
/* The same on NV12 device planes (laid out as in mc_process_clip_nv12_device; channels is 3).  For any NV12
 * input X it equals mc_chain_process_device on cv2.cvtColor(X, COLOR_YUV2BGR_NV12): the same bytes written, flags, info
 * and state.  The front converts each source pixel inside its tap walk, so no full-resolution BGR frame is stored.  The
 * outputs are BGR or gray, not NV12 (a cropped or downscaled frame may have odd dimensions); with grayscale on this is
 * gray magnification of an NV12 source.  The NV12 checks of mc_process_nv12_device apply to `in` (width and height
 * even and >= 2, pitch >= width, lane_stride >= pitch * height with more than one virtual lane). */
mc_status mc_chain_process_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                       const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                       uint8_t* d_original, size_t original_step, uint8_t* produced, mc_chain_info* info);

/* --- the export canvas on the device (SURVEY.md 8f-2) -------------------------------------------------------------
 * The frame the reference's exporter writes to the file, compose(original, cur, split) of src/export/Exporter.cpp:25-34,
 * 53-88 (its labels through mc_set_overlay, below): both taps are expanded to BGR (a gray frame as GRAY2BGR) and cropped, from the top-left
 * corner, to their common even size w x h (W & ~1, H & ~1 of the chain's output, which H.264 / FFV1 need); then
 *   MC_SPLIT_NONE        the processed pane alone: w x h
 *   MC_SPLIT_LEFT_RIGHT  the original pane left of the processed one: 2w x h
 *   MC_SPLIT_TOP_BOTTOM  the original pane above the processed one: w x 2h
 * A canvas is packed BGR (pitch >= 3 * its width), NV12 (pitch >= its width; cvtColor(COLOR_BGR2YUV_I420) of the BGR
 * canvas with Cb,Cr interleaved, as the NV12 calls write) or I420 (the planes cvtColor(COLOR_BGR2YUV_I420) returns; see
 * the planar 4:2:0 section), or RGB: packed R,G,B (MC_CANVAS_RGB, pitch >= 3 * its width) or three planes R, G, B
 * (MC_CANVAS_RGB_PLANAR; see the RGB section).  Its dimensions are always even, so a 4:2:0 canvas always exists when the
 * BGR one does. */
typedef enum mc_split { MC_SPLIT_NONE = 0, MC_SPLIT_LEFT_RIGHT = 1, MC_SPLIT_TOP_BOTTOM = 2 } mc_split; /* livim::SplitMode */
typedef enum mc_canvas_format {
    MC_CANVAS_BGR = 0, MC_CANVAS_NV12 = 1, MC_CANVAS_I420 = 2, MC_CANVAS_RGB = 3, MC_CANVAS_RGB_PLANAR = 4
} mc_canvas_format;
typedef struct mc_canvas {
    int32_t format;       /* mc_canvas_format */
    uint8_t* data;        /* BGR / RGB: canvas of virtual lane 0; NV12 / I420: its luma plane; RGB_PLANAR: its R plane,
                             with the G and B planes at data + pitch * canvas_h and data + 2 * pitch * canvas_h */
    uint8_t* uv;          /* NV12: interleaved Cb,Cr plane (need not follow the luma); I420: Cb plane, with the Cr plane
                             at uv + (pitch / 2) * (canvas_h / 2); BGR, RGB, RGB_PLANAR: unused */
    size_t pitch;         /* bytes per row (both NV12 planes; the I420 luma plane, whose chroma rows are pitch / 2 apart;
                             each RGB_PLANAR plane) */
    size_t lane_stride;   /* bytes from one virtual lane's canvas (planes) to the next */
} mc_canvas;

/* Canvas size compose() gives the chain's output of a width x height x channels frame (no handle, no GPU); 0 x 0 when a
 * pane would be empty (the reference skips that frame).  MC_ERR_INVALID when p or an output is NULL, the split is out
 * of range or channels is not 1 or 3. */
mc_status mc_compose_geometry(const mc_params* p, int width, int height, int channels, int grayscale, int split,
                              int* canvas_w, int* canvas_h);

/* mc_chain_process_device / mc_chain_process_nv12_device followed by compose(original, cur, split) for every virtual
 * lane v = t * lanes + k, whose canvas is at v * lane_stride of the canvas planes:
 *   The produced flags, info, the temporal state afterwards and mc_lane_produced are exactly those of the chain call.
 *   The canvas of every virtual lane that is not held is written, whether the magnifier produced or not (the exporter
 *   writes a frame every step): `cur` is then the front's output, or the input when no front stage runs.  Held lanes,
 *   row padding, and every canvas of a 0 x 0 geometry are left untouched.
 *   The original pane is the preprocessed frame when a Preprocess stage runs, otherwise the input; an NV12 input is read
 *   through its BGR conversion, so the NV12 call equals the BGR call on cv2.cvtColor(X, COLOR_YUV2BGR_NV12).
 *   One "compose" kernel (profile_kernels) writes every canvas straight from the taps: gray and NV12 sources are
 *   converted in registers, and no full-resolution BGR frame is stored for them.
 *   Errors, returned before any kernel runs and with no canvas or state changed: MC_ERR_INVALID for a split out of
 *   range, a NULL canvas or canvas plane, a pitch smaller than a canvas row, lane_stride < pitch * canvas height with
 *   more than one virtual lane, a canvas that is not 0 x 0 and not the geometry of the overlay set (mc_set_overlay),
 *   and the chain call's own argument errors (d_out / d_original are not arguments here).
 *   Device scratch: besides the chain's, the magnifier's output for the largest frame set seen (out_w * out_h *
 *   out_channels bytes per virtual lane), a byte per virtual lane for the pane choice, and, with a split and a
 *   Preprocess stage, the preprocessed frames in the front's staging. */
mc_status mc_chain_compose_device(mc_handle* h, const uint8_t* d_in, int frames, int width, int height, int channels,
                                  size_t in_step, const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                  uint8_t* produced, mc_chain_info* info);
mc_status mc_chain_compose_nv12_device(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                       const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                       uint8_t* produced, mc_chain_info* info);

/* --- labels on the export canvas (ExportRequest::textOverlay, Exporter.cpp:36-50) ------------------------------------
 * The exporter's "Original" / "Processed" labels darken a box (addWeighted(box, 0.35, black, 0.65, 0)) and draw white
 * anti-aliased text over it.  Both steps are pointwise and treat the three channels alike, so a labelled canvas is
 *     out[y][x][c] = map[index(x, y)][in[y][x][c]]
 * inside a few rectangles and the canvas itself outside them: one u8 -> u8 tone map per labelled pixel.  The caller
 * builds these maps once per export geometry by drawing the labels with its own OpenCV onto the 256 flat grey canvases
 * (live-video-magnification_b200/labels.py is the executable specification; INTEGRATION.md §2b), and the compose
 * kernel applies them to every canvas it writes.  The core draws no text itself.
 *   Configuration, not temporal state: the overlay belongs to the handle and is kept across mc_reset, structural
 *     resets and failed frames, until it is replaced or cleared.
 *   Stream order: mc_set_overlay copies the overlay to device memory in stream order on mc_stream().  Compose calls
 *     enqueued before it use the previous overlay, calls after it the new one.  The caller's buffers may be freed as
 *     soon as it returns.
 *   Every compose call (BGR, NV12, YUYV, I420 and RGB sources; BGR, NV12, I420 and RGB canvases; frames, clips and lanes)
 *     maps each canvas it writes: a canvas pixel inside a rect becomes map[index][v] in each of its channels, before the
 *     4:2:0 conversion or the RGB channel order (a
 *     2x2 block whose top-left pixel is labelled takes its Cb,Cr from the labelled value).  Held lanes and 0 x 0
 *     canvases stay untouched, as without an overlay.  Chain calls that do not compose ignore it.
 *   Errors, MC_ERR_INVALID: mc_set_overlay with canvas_w or canvas_h < 1, rects or maps out of range, a NULL map or
 *     index, a rect that is empty or not inside the canvas, two rects that overlap, or an index >= maps; the previous
 *     overlay is kept.  A compose call while an overlay is set whose canvas (mc_compose_geometry) is neither 0 x 0 nor
 *     canvas_w x canvas_h, returned before any kernel runs with no canvas or state changed: a stale overlay is never
 *     dropped or misplaced silently.
 *   Device memory: maps * 256 bytes plus 2 bytes per rect pixel, kept for the largest overlay set. */
#define MC_OVERLAY_MAX_RECTS 2
typedef struct mc_overlay_rect {
    int32_t x, y, w, h;          /* on the canvas, inside it */
    const uint16_t* index;       /* host: h rows of w entries, the tone map of each pixel */
} mc_overlay_rect;
typedef struct mc_overlay {
    int32_t canvas_w, canvas_h;                 /* the canvas geometry it was built for */
    int32_t rects;                              /* 0 .. MC_OVERLAY_MAX_RECTS, pairwise disjoint */
    mc_overlay_rect rect[MC_OVERLAY_MAX_RECTS];
    int32_t maps;                               /* 1 .. 65536 */
    const uint8_t* map;                         /* host: maps x 256 bytes, map[m][v] */
} mc_overlay;
/* Sets the handle's overlay (see above); ov == NULL clears it. */
mc_status mc_set_overlay(mc_handle* h, const mc_overlay* ov);

/* --- packed 4:2:2 camera frames (V4L2 YUYV / UYVY) into the processing chain ---------------------------------------
 * A YUYV frame is height rows of width / 2 groups of 4 bytes, Y0 Cb Y1 Cr (UYVY: Cb Y0 Cr Y1); both pixels of a group
 * take its Cb,Cr.  The core converts it exactly as OpenCV's capture does, cvtColor(COLOR_YUV2BGR_YUYV / _UYVY) (BT.601
 * limited range, the fixed point of the NV12 conversion), pixel by pixel inside the chain's front kernel, so no
 * full-resolution BGR frame is stored unless the caller asks for it.
 *   Equivalence: for any input X, a call equals the BGR chain call (mc_chain_process_device / _compose_device /
 *     mc_chain_process, channels 3) on B = cv2.cvtColor(X, COLOR_YUV2BGR_YUYV or _UYVY), bit for bit: the processed
 *     frames, the original tap, the produced flags, mc_lane_produced and the temporal state afterwards.  YUYV, NV12 and
 *     BGR calls of the same geometry interleave on one handle without a structural reset (the tracker sees channels 3).
 *   The conversion is a front stage that always runs: where the BGR call would leave its result to the input
 *     (cur_is_input / orig_is_input), the YUYV call writes it, B or its BGR2GRAY under grayscale.  `info` has
 *     cur_is_input = orig_is_input = 0, and the geometry of the front's output (width x height without a Preprocess
 *     stage).  d_out is written for every virtual lane that is not held, and so is d_original when it is not NULL.
 *   Compose: the original pane is the preprocessed frame when a Preprocess stage runs, otherwise B, read straight from
 *     the YUYV frame.
 *   Errors: MC_ERR_INVALID, before any kernel or copy runs and with no caller buffer or state changed, for a NULL `in` or
 *     `data`, an order out of range, width odd or < 2, height < 1, pitch < 2 * width, lane_stride < pitch * height with
 *     more than one virtual lane, and every argument error of the matching BGR call.  Held lanes, Color's multi-lane
 *     refusals (MC_ERR_UNSUPPORTED) and the clip rules are those of the BGR calls.
 *   Device scratch: the front's staging holds B (width x height x 3 per virtual lane) when neither d_original nor a
 *     gray-only magnifier input takes its place. */
typedef enum mc_yuv422_order { MC_YUV422_YUYV = 0, MC_YUV422_UYVY = 1 } mc_yuv422_order;
typedef struct mc_yuv422 {
    uint8_t* data;        /* frame of (virtual) lane 0: height rows of 2 * width bytes */
    size_t pitch;         /* bytes per row (V4L2 bytesperline), >= 2 * width */
    size_t lane_stride;   /* bytes from one virtual lane's frame to the next */
    int32_t order;        /* mc_yuv422_order */
} mc_yuv422;

/* device frames, every lane, clips: the layout and rules of mc_chain_process_nv12_device (frame t of lane k is virtual
 * lane t * lanes + k, at v * lane_stride of `data`) */
mc_status mc_chain_process_yuv422_device(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                         const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                         uint8_t* d_original, size_t original_step, uint8_t* produced, mc_chain_info* info);
/* the same followed by compose (export from a YUYV recording): the rules of mc_chain_compose_nv12_device */
mc_status mc_chain_compose_yuv422_device(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                         const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                         uint8_t* produced, mc_chain_info* info);
/* the live camera form: one host frame (pinned or pageable), 1-lane handle, blocking; the rules of mc_chain_process.
 * Only the 2 * width bytes of each row cross PCIe (2 B/px against 3 for BGR).  `out` and `original` (either may be
 * NULL) are written tight; out_bytes / original_bytes smaller than info's frames are MC_ERR_INVALID before any copy. */
mc_status mc_chain_process_yuv422(mc_handle* h, const mc_yuv422* in, int width, int height, const mc_params* p,
                                  int grayscale, uint8_t* out, size_t out_bytes, uint8_t* original, size_t original_bytes,
                                  mc_chain_info* info);
/* mc_chain_submit on packed 4:2:2 host frames (the checks of mc_chain_process_yuv422_device): 2 B/px cross PCIe upwards,
 * and both frames come back, as every chain call on a 4:2:2 source writes them. */
mc_status mc_chain_submit_yuv422(mc_handle* h, const mc_yuv422* in, int width, int height, const mc_params* p, int grayscale,
                                 uint8_t* out, size_t out_step, uint8_t* original, size_t original_step, mc_chain_info* info);

/* --- the export canvas from host clips, pipelined (an exporter that decodes to host memory) ---------------------------
 * mc_chain_compose_device / _nv12_device / _yuv422_device on host memory, submitted and collected as mc_submit is: one
 * call submits a clip of `frames` consecutive frames of every lane, and mc_collect collects it, in strict FIFO order with
 * mc_submit, mc_submit_nv12, the chain submits and the other compose submits on the handle.  An exporter submits T decoded
 * frames and collects T finished canvases in file order, with the uploads, kernels and downloads of up to
 * mc_pipeline_depth() clips overlapped.
 *   Memory: `in` and `canvas` have the layout of the matching device compose call, on host memory: virtual lane
 *     v = t * lanes + k has its input at v * height * in_step (NV12 and 4:2:2 frames: at v * lane_stride) and its canvas
 *     (BGR, or both NV12 planes) at v * canvas->lane_stride.  Each buffer may be pinned or pageable, independently of the
 *     others.  All of them must stay valid until the submit is collected, and `in` must also stay unchanged until then.
 *   Equivalence: for any sequence of compose submits, with restarts, holds, mc_set_lane_params, mc_set_overlay, parameter,
 *     ROI or levels changes between them and mixed with the other submits, every byte of every canvas, the produced
 *     flags, mc_lane_produced and the temporal state after each collect equal, bit for bit, those of the matching device
 *     compose call on the same frames uploaded by the caller.  Lifecycle, lane parameters and the overlay are taken at
 *     submit (for a clip, at its first frame, as in the device clip calls); frames in flight keep what they were
 *     submitted with.
 *   What is written: that of the device compose call.  The canvas of every virtual lane that is not held is downloaded;
 *     held lanes, row padding and the canvases of a 0 x 0 geometry are left untouched.
 *   produced: frames * lanes host bytes, [t][lane], written by the mc_collect that collects the submit, and valid until
 *     then.  *produced of that mc_collect is "at least one virtual lane produced"; mc_lane_produced then reports the
 *     flags of the clip's last frame (a submit does not change it before it is collected).
 *   info: filled by the submit, final when it returns, with magnified 0 (the collected flags carry that fact).
 *   Errors, returned before any copy or kernel is enqueued, with the handle's state and the frames in flight unchanged:
 *     MC_ERR_INVALID for every argument error of the matching device compose call (overlay geometry included): frames <
 *     1, frames * lanes > MC_MAX_LANES and a NULL produced among them; for a full pipeline; and for slot buffers that
 *     would have to grow while frames are in flight ("pipeline geometry changed").  MC_ERR_UNSUPPORTED for Color's
 *     multi-lane refusals.  The device clip calls keep refusing while submitted frames are in flight.
 *   Memory per pipeline slot (mc_pipeline_depth() slots, each grown, never shrunk, only while nothing is in flight):
 *     device memory for the clip's input (frames * lanes * its bytes per frame: width * height * channels, NV12 1.5 and
 *     4:2:2 2 bytes per pixel) and for the canvases of this frame size and split without a crop or downscale (frames *
 *     lanes * cw * ch * 3 bytes for BGR, * 1.5 for NV12 canvases), so that a ROI or downscale change and an export's
 *     last, shorter clip fit in the slots that are there.  At T = 16, 1080p BGR in and a left/right BGR canvas that is
 *     about 100 MB in plus 200 MB out per slot.  Pinned host staging for a submit's input or canvas bytes is allocated
 *     (per slot, grow-only) only when that buffer is pageable; pinned buffers are copied straight to and from device
 *     memory, and pageable ones cost two host copies of every byte on the calling thread. */
mc_status mc_chain_compose_submit(mc_handle* h, const uint8_t* in, int frames, int width, int height, int channels,
                                  size_t in_step, const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                  uint8_t* produced, mc_chain_info* info);
mc_status mc_chain_compose_submit_nv12(mc_handle* h, const mc_nv12* in, int frames, int width, int height,
                                       const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                       uint8_t* produced, mc_chain_info* info);
mc_status mc_chain_compose_submit_yuv422(mc_handle* h, const mc_yuv422* in, int frames, int width, int height,
                                         const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                         uint8_t* produced, mc_chain_info* info);

/* --- planar 4:2:0 frames (I420 / YV12): the hand-off format of software decoders and encoders -------------------------
 * FFmpeg's software decoders and encoders (libx264, FFV1, MJPEG; AV_PIX_FMT_YUV420P) and cv::VideoCapture / VideoWriter
 * exchange 4:2:0 YCbCr in three planes: a luma plane and a Cb and a Cr plane of height/2 rows of width/2 bytes, one Cb and
 * one Cr per 2x2 pixel block.  BT.601 limited range, as NV12: OpenCV converts I420 and YV12 with the fixed point of its
 * NV12 conversion, and the core converts them on the device with the same arithmetic.
 *   Equivalence, input: let X be any I420 input.  Every call on X equals, bit for bit, the NV12 call on the frame with X's
 *     Y plane and its U, V planes interleaved, and therefore the BGR call on cv2.cvtColor(X, COLOR_YUV2BGR_I420) (_YV12
 *     when the planes are YV12's): the processed frames, the original tap, `info`, the produced flags, mc_lane_produced
 *     and the temporal state afterwards.  I420, NV12, 4:2:2 and BGR calls of the same geometry interleave on one handle
 *     without a structural reset (the tracker sees channels 3).  A ROI at an odd column or row still takes each pixel's
 *     chroma from its own 2x2 block of the frame.
 *   Equivalence, canvas: an MC_CANVAS_I420 canvas's Y, Cb and Cr planes equal the NV12 canvas of the same call with its
 *     chroma de-interleaved, which is cv2.cvtColor(bgr_canvas, COLOR_BGR2YUV_I420), labels included (a 2x2 block whose
 *     top-left pixel is labelled takes its Cb,Cr from the labelled value).  Every compose call accepts it: BGR, gray,
 *     NV12, 4:2:2 and I420 sources; device and submit; frames, clips and lanes.  Held lanes, 0 x 0 canvases and row
 *     padding stay untouched, the bytes between canvas_w / 2 and pitch / 2 of each chroma row included.  The layout is
 *     that of av_image_alloc / x264_picture_alloc buffers whose chroma linesize is half the luma's.
 *   Errors, returned before any kernel or copy runs, with no caller buffer, state or frame in flight changed:
 *     MC_ERR_INVALID for a NULL descriptor or plane, width or height odd or < 2, pitch < width, chroma_pitch < width / 2,
 *     lane_stride < pitch * height with more than one virtual lane, and every argument error of the NV12 twin.  An I420
 *     canvas: MC_ERR_INVALID for a NULL data or uv, an odd pitch or pitch < canvas_w.
 *   Memory: staging and pipeline slots follow the NV12 rules, 1.5 B/px for frames and canvases.  Pageable planes go
 *     through pinned staging; pinned planes are copied directly. */
typedef struct mc_yuv420p {
    uint8_t* y;            /* luma plane of (virtual) lane 0: height rows of width bytes */
    uint8_t* u;            /* Cb plane: height/2 rows of width/2 bytes */
    uint8_t* v;            /* Cr plane: height/2 rows of width/2 bytes; YV12 is passed with u / v at its Cb / Cr planes */
    size_t pitch;          /* luma bytes per row (AVFrame linesize[0]) */
    size_t chroma_pitch;   /* Cb and Cr bytes per row (linesize[1] == linesize[2]) */
    size_t lane_stride;    /* bytes from one virtual lane's planes to the next, the same for all three */
} mc_yuv420p;
/* mc_chain_process_nv12_device on I420 device planes (frame t of lane k is virtual lane t * lanes + k) */
mc_status mc_chain_process_yuv420p_device(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                          const mc_params* p, int grayscale, uint8_t* d_out, size_t out_step,
                                          uint8_t* d_original, size_t original_step, uint8_t* produced, mc_chain_info* info);
/* mc_chain_compose_nv12_device on I420 device planes */
mc_status mc_chain_compose_yuv420p_device(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                          const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                          uint8_t* produced, mc_chain_info* info);
/* mc_chain_submit_nv12 on I420 host planes: 1.5 B/px cross PCIe upwards */
mc_status mc_chain_submit_yuv420p(mc_handle* h, const mc_yuv420p* in, int width, int height, const mc_params* p, int grayscale,
                                  uint8_t* out, size_t out_step, uint8_t* original, size_t original_step, mc_chain_info* info);
/* mc_chain_compose_submit_nv12 on I420 host planes: an exporter that decodes and encodes I420 in software submits its
 * decoded frames and collects canvases its encoder takes as they are */
mc_status mc_chain_compose_submit_yuv420p(mc_handle* h, const mc_yuv420p* in, int frames, int width, int height,
                                          const mc_params* p, int grayscale, int split, const mc_canvas* canvas,
                                          uint8_t* produced, mc_chain_info* info);

/* --- RGB frames (packed RGB, RGBA / BGRA, planar RGB): PyTorch tensors, Python image libraries and desktop capture ------
 * torchvision's decode_jpeg(device="cuda") returns planar RGB (3, H, W) u8 tensors and image models take (N, 3, H, W)
 * batches; PyAV's to_ndarray(format="rgb24"), PIL and imageio hand out packed RGB; desktop and GPU capture (Media
 * Foundation RGB32, CoreVideo 32BGRA, GStreamer BGRx / RGBA, GL readbacks) hand out 32-bit BGRA / RGBA pixels.  The core
 * reads every such frame where it is and swaps its channels on the device.
 *   Equivalence, input: let X be any RGB input and B = cv2.cvtColor(X, COLOR_RGB2BGR / COLOR_RGBA2BGR / COLOR_BGRA2BGR)
 *     (planar X: cv2.merge([B_plane, G_plane, R_plane])).  Every call on X equals, bit for bit, the BGR call on B: the
 *     processed frames, the original tap, the produced flags, mc_lane_produced and the temporal state afterwards.  The
 *     conversion is a front stage that always runs, as for 4:2:2: `info` has cur_is_input = orig_is_input = 0, and
 *     d_out / d_original receive B (or its BGR2GRAY under grayscale) where a BGR call would leave the result to the
 *     input.  RGB, BGR, NV12, 4:2:2 and I420 calls of one geometry interleave on a handle without a structural reset
 *     (the tracker sees channels 3).  The 4th byte of an RGBA / BGRA pixel is never read.
 *   Equivalence, canvas: an MC_CANVAS_RGB canvas is cv2.cvtColor(bgr_canvas, COLOR_BGR2RGB) of the BGR canvas of the
 *     same call, labels included (the overlay's tone maps act on each channel alike); an MC_CANVAS_RGB_PLANAR canvas is
 *     that BGR canvas's channels 2, 1, 0 as planes, one CHW tensor per virtual lane.  Every compose call accepts both:
 *     BGR, gray, NV12, 4:2:2, I420 and RGB sources; device and submit; frames, clips and lanes.  Held lanes, 0 x 0
 *     canvases, row padding and the padding after each plane stay untouched.
 *   Errors, returned before any kernel or copy runs, with no caller buffer, state or frame in flight changed:
 *     MC_ERR_INVALID for a NULL descriptor, data or (planar) g / b, a layout out of range, width or height < 1, pitch <
 *     width * bytes per pixel (planar: < width), lane_stride < pitch * height with more than one virtual lane, and every
 *     argument error of the BGR twin.  An RGB canvas: MC_ERR_INVALID for a NULL data, pitch < 3 * canvas_w (planar: <
 *     canvas_w) and, with more than one virtual lane, lane_stride < pitch * canvas_h (planar: < 3 * pitch * canvas_h).
 *     Color's multi-lane refusals stay MC_ERR_UNSUPPORTED.
 *   Memory: only width * bytes per pixel of each row crosses PCIe (3 B/px; RGBA / BGRA 4 B/px), and canvases come back
 *     at 3 B/px.  Pageable frames go through pinned staging; pinned ones are copied directly. */
typedef enum mc_rgb_layout {
    MC_RGB_RGB = 0,      /* packed R,G,B, 3 bytes per pixel (rgb24, HWC RGB arrays and tensors) */
    MC_RGB_RGBA = 1,     /* packed R,G,B,A (or X), 4 bytes per pixel; the 4th byte is never read */
    MC_RGB_BGRA = 2,     /* packed B,G,R,A (or X), 4 bytes per pixel; the 4th byte is never read */
    MC_RGB_PLANAR = 3    /* three planes R, G, B of width bytes per row (CHW / NCHW tensors) */
} mc_rgb_layout;
typedef struct mc_rgb {
    uint8_t* data;        /* packed: frame of (virtual) lane 0; planar: its R plane */
    uint8_t* g;           /* planar: G plane; packed: unused */
    uint8_t* b;           /* planar: B plane; packed: unused */
    size_t pitch;         /* bytes per row (every plane) */
    size_t lane_stride;   /* bytes from one virtual lane's frame (planes) to the next */
    int32_t layout;       /* mc_rgb_layout */
} mc_rgb;
/* mc_chain_process_device on RGB device frames (frame t of lane k is virtual lane t * lanes + k) */
mc_status mc_chain_process_rgb_device(mc_handle* h, const mc_rgb* in, int frames, int width, int height, const mc_params* p,
                                      int grayscale, uint8_t* d_out, size_t out_step, uint8_t* d_original,
                                      size_t original_step, uint8_t* produced, mc_chain_info* info);
/* mc_chain_compose_device on RGB device frames: e.g. the planes of an (N, 3, H, W) CUDA tensor in, planar RGB canvases
 * of another tensor out */
mc_status mc_chain_compose_rgb_device(mc_handle* h, const mc_rgb* in, int frames, int width, int height, const mc_params* p,
                                      int grayscale, int split, const mc_canvas* canvas, uint8_t* produced,
                                      mc_chain_info* info);
/* mc_chain_submit on RGB host frames */
mc_status mc_chain_submit_rgb(mc_handle* h, const mc_rgb* in, int width, int height, const mc_params* p, int grayscale,
                              uint8_t* out, size_t out_step, uint8_t* original, size_t original_step, mc_chain_info* info);
/* mc_chain_compose_submit on RGB host frames: an exporter that decodes rgb24 or captures BGRA submits its frames as
 * they are */
mc_status mc_chain_compose_submit_rgb(mc_handle* h, const mc_rgb* in, int frames, int width, int height, const mc_params* p,
                                      int grayscale, int split, const mc_canvas* canvas, uint8_t* produced,
                                      mc_chain_info* info);

/* Pinned host memory for frames (so FramePool buffers can be DMA'd directly). */
void* mc_host_alloc(size_t bytes);
void mc_host_free(void* p);

/* The handle's cudaStream_t (as void*) so callers can order their own work / record events on it. */
void* mc_stream(mc_handle* h);

/* Options (call before the first frame or after mc_reset):
 *   "faithful_level0" (default 0): also run the level-0 band + IIR state update that the reference
 *        performs although the gain loop multiplies that band by 0 (MagnifyCore.hpp:130-131); needed
 *        only to compare level-0 state planes with the oracle.
 *   "pipeline_depth"  (default 3)
 *   "keep_float_output" (default 0): keep the pre-quantisation float image (tests)
 *   "profile_kernels" (default 0): see mc_profile_read
 *   "use_tma" (default 1): stage the fused level kernel's tiles with TMA (cp.async.bulk.tensor): its input window and
 *        the tile's two state planes are requested at kernel entry; 0 selects the 128-bit LDG staging path that also
 *        runs when a tensor map cannot be encoded (same results)
 *   "lane_groups" (default 0 = automatic: min(2, lanes / 8), at least 1): Laplace — the lanes of the handle run as
 *        that many concurrent launch chains on separate CUDA streams, forked from and joined into mc_stream(); the
 *        L1-bound ingest, issue-bound egress and HBM-bound level kernels of different groups then share the SMs
 *        instead of running back to back (same results; profile_kernels forces 1)
 *   "egress_strip" (default 1): Laplace egress runs as the shuffle strip kernel (one warp per 128-column strip,
 *        sliding windows in per-lane shared-memory rings); 0 selects the shared-memory tile kernel, the reference the
 *        strip kernel is tested against (bit-identical results); any non-zero value selects the strip kernel
 *   "analysis_only" (default 0): Laplace and Phase — frames after the first update the temporal state (EMA planes;
 *        Riesz pyramids, phase accumulators and Butterworth registers) but skip synthesis and egress and report
 *        *produced = 0; the cheap first pass of temporal sharding (SURVEY 8f-3)
 *   "band_from_state" (default 1): Laplace synthesis rebuilds each amplified band gain*(hi-lo) from the two
 *        state planes instead of reading a band plane stored by the level kernel (same results; takes 4 B/px off
 *        the level kernel's interface and adds them to the collapse / egress kernels; 0 kept for A/B measurements)
 *   "color_lane_lifecycle" (default 0): Color on a handle with lanes > 1 accepts mc_hold_lane and single-lane
 *        mc_restart_lane (see the lane lifecycle above) instead of refusing them with MC_ERR_UNSUPPORTED; lanes that
 *        run in lock-step give the same results either way */
mc_status mc_set_option(mc_handle* h, const char* key, int value);

/* Test-only access to temporal state planes as dense f32 [lanes][channels][rows][cols].
 * Names: Laplace "lowpassHi" / "lowpassLo" (MotionState, MagnifyCore.hpp:24-29), level 0..levels (levels 0 and
 *   `levels` exist only with option faithful_level0); Laplace "band", the frame path's band planes of a level: the
 *   amplified band gain * (hi - lo) the level kernel stores (levels 1..levels-1 with band_from_state 0), overwritten by
 *   the collapse sum cur_l at levels 2..levels-2 (so on a frame that synthesised, "band" at levels 2..levels-2 is
 *   cur_l, not the band).  When a frame synthesises L only (zero chroma, see DESIGN.md §4) their a / b planes are
 *   left as they are;
 * Laplace, read-only (mc_set_state returns MC_ERR_INVALID): "gauss", level 1..levels, the Gaussian pyramid G_l of the
 *   last frame call, `channels` channels.  It follows "lab16": it exists only after a frame call, and is absent before
 *   the first frame, after mc_reset, after a clip call (clips build their own pyramid) and after a change of mode or
 *   geometry; for gray input it exists as well.  It is absent when levels is 1 without faithful_level0, where no
 *   kernel builds G_1.  A held lane keeps in it what an earlier frame left;
 * Phase, per band level 0..levels-2, one channel: "old.lowpass", "old.rx", "old.ry" (RieszState::old),
 *   "phase.c", "phase.s" (itsPhase — the two filters' copies are identical), "lo.r0.c", "lo.r0.s", "lo.r1.c",
 *   "lo.r1.s", "hi.r0.c", "hi.r0.s", "hi.r1.c", "hi.r1.s" (itsRegister0/1 of the low / high cutoff filters,
 *   TemporalFilter.cpp:299-317);
 * Phase, read-only (mc_set_state returns MC_ERR_INVALID), the buffers of the last frame call, one channel:
 *   "oct", level 0..levels-1: octave i of the analysis (level 0 the f32 L plane, level levels-1 the residual the collapse
 *   starts from); "amp", "t_c", "t_s", band level 0..levels-2: the phase kernel's amplitude and (hiIIR - loIIR) *
 *   amplitude; "amplified", band level 0..levels-2: the amplified band; "collapsed", band level 0..levels-2: the
 *   collapse result of that level (level 0 is the L' the egress merges with a, b).  They follow "lab16": they exist only
 *   after a frame call on 3-channel input, and are absent before the first frame, after mc_reset, after a clip call and
 *   after a change of mode or geometry.  "amp" / "t_c" / "t_s" exist only when some lane ran the phase kernel (not on a
 *   frame where every lane is on its first frame or held), "amplified" / "collapsed" only when the frame was amplified
 *   (not under analysis_only).  A lane that did not run (first frame, held) keeps in them what an earlier frame left;
 *   a held lane also keeps its "oct".
 * Color, read-only (mc_set_state returns MC_ERR_INVALID), the buffers of the last frame call, `channels` channels:
 *   "gauss", level 0..levels: the Gaussian pyramid (level 0 is the u8 frame as f32);
 *   "window", level k = logical column 0..n-1 of the rolling window (column 0 the oldest), each lane's own ring slot,
 *   as rows x cols of the smallest pyramid level;
 *   "filtered", level k: the same column after the inverse DFT, before normalisation (both DFT scales applied);
 *   "up", level 0..levels (+1 when the bilinear resize ran): level 0 is the normalised reconstructed column times the
 *   amplification, the last level the colour image that is added to the input.
 *   Lanes of one handle may have windows of different length: a column is served only while every lane has it, and
 *   "filtered" / "up" only while every lane ran the filter in the last frame call that was not held for all lanes
 *   (otherwise 0 rows).  A held lane's "gauss" is the pyramid of whatever its input slot held (in a chain call with
 *   a front stage, which skips held lanes, bytes an earlier call left in the front's staging).  All are absent before the first frame and after mc_reset or a change of mode or geometry.
 * Laplace and Phase, level 0, three channels, read-only: "lab16", the BGR->Lab conversion of the last frame call as
 *   the kernels hold it, the raw fixed-point values L*2^14/100, (a+128)*64, (b+128)*64 widened (exactly) to f32.  It
 *   exists only after a frame call on 3-channel input; before the first frame, after mc_reset and after a clip call it
 *   is absent (clips convert into their own scratch).  A held lane keeps the planes of its last converted frame.
 *   mc_set_state on it returns MC_ERR_INVALID.
 * mc_state_dims reports rows/cols/channels for a name+level (0 rows if absent). */
mc_status mc_state_dims(mc_handle* h, const char* name, int level, int* rows, int* cols, int* channels);
mc_status mc_get_state(mc_handle* h, const char* name, int level, float* dst, size_t dst_floats);
mc_status mc_set_state(mc_handle* h, const char* name, int level, const float* src, size_t src_floats);

/* Debug tap: last frame's pre-quantisation BGR/gray float output in [0,1] ([lanes][rows][cols][C]);
 * enabled by option "keep_float_output" = 1. */
mc_status mc_get_float_output(mc_handle* h, float* dst, size_t dst_floats);

/* Number of kernel launches this handle has issued (for bench.py's gpu_launches). */
uint64_t mc_launch_count(mc_handle* h);

/* Per-kernel device timing for bench.py's roofline: with option "profile_kernels" = 1 every launch
 * is bracketed by CUDA events on the handle's stream.  mc_profile_read synchronises, drains them and
 * writes text lines "kernel level launches total_ms\n" (NUL-terminated) into buf. */
mc_status mc_profile_read(mc_handle* h, char* buf, size_t cap);

/* Last error text for this handle (or for a failed mc_create when h == NULL); never NULL. */
const char* mc_last_error(mc_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* MAGCORE_B200_H */
