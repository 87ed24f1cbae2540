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
 *   Color:   one frame call per frame (same results; the clip call works whatever the mode).
 * MC_ERR_INVALID, with the state untouched, when frames < 1, frames * lanes > MC_MAX_LANES, produced is NULL or frames of
 * mc_submit are in flight; the parameter checks of mc_process_device apply unchanged.  Mode None and an empty image
 * are the identity (all flags 0, state dropped).  A failed clip drops the state like a failed frame.  The clip path
 * keeps device scratch for the largest clip seen, released by mc_reset: ~29 MB (Laplace) or ~82 MB (Phase) per 1080p
 * colour frame at 6 levels. */
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
 *     > 1 follows the clip rules of mc_process_clip_device unchanged (lifecycle taken at the first frame, Laplace and
 *     Phase batched, Color a loop of frame calls).
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
 *     frames * lanes > MC_MAX_LANES, NULL produced / info / params, or frames of mc_submit in flight; MC_ERR_UNSUPPORTED
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
 *   "use_tma" (default 1): stage the fused level kernel's tiles with TMA (cp.async.bulk.tensor); 0 selects
 *        the 128-bit LDG staging path (same results; kept for A/B measurements)
 *   "prefetch_state" (default 1; needs use_tma): the fused level kernel requests the tile's two state planes as TMA
 *        bulk copies at kernel entry, together with its input window, instead of loading them in its last phase
 *        (same results; 0 kept for A/B measurements)
 *   "lane_groups" (default 0 = automatic: min(2, lanes / 8), at least 1): Laplace — the lanes of the handle run as
 *        that many concurrent launch chains on separate CUDA streams, forked from and joined into mc_stream(); the
 *        L1-bound ingest, issue-bound egress and HBM-bound level kernels of different groups then share the SMs
 *        instead of running back to back (same results; profile_kernels forces 1)
 *   "egress_strip" (default 16): Laplace egress runs as the shuffle strip kernel (one warp per 128-column strip,
 *        sliding windows in per-lane shared-memory rings; the value 16 / 20 / 24 picks the register cap = resident
 *        warps per SM, 1 means the default); 0 selects the shared-memory tile kernel (bit-identical results; kept for A/B)
 *   "ingest_warps" (default 1): warps per CTA (1, 2 or 4) of the fused BGR->Lab ingest kernel (same results; A/B)
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
 *   the collapse sum cur_l at levels 2..levels-2.  When a frame synthesises L only (zero chroma, see DESIGN.md
 *   §4) their a / b planes are left as they are;
 * Phase, per band level 0..levels-2, one channel: "old.lowpass", "old.rx", "old.ry" (RieszState::old),
 *   "phase.c", "phase.s" (itsPhase — the two filters' copies are identical), "lo.r0.c", "lo.r0.s", "lo.r1.c",
 *   "lo.r1.s", "hi.r0.c", "hi.r0.s", "hi.r1.c", "hi.r1.s" (itsRegister0/1 of the low / high cutoff filters,
 *   TemporalFilter.cpp:299-317);
 * Color keeps its rolling window in a device ring buffer that is not exposed.
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
