// Motion (Laplace) per-frame driver — device twin of magcore::magnifyMotion
// (reference src/processing/magnification/MagnifyCore.hpp:83-160).
#include <algorithm>
#include <cstring>

#include "mc_modes.h"

namespace mc {

cudaError_t DeviceArena::alloc(float** p, size_t floats) {
    void* v = nullptr;
    cudaError_t e = alloc_bytes(&v, floats * sizeof(float));
    *p = (float*)v;
    return e;
}
cudaError_t DeviceArena::alloc_bytes(void** p, size_t bytes) {
    *p = nullptr;
    cudaError_t e = cudaMalloc(p, bytes ? bytes : 4);
    if (e == cudaSuccess) blocks.push_back(*p);
    return e;
}
void DeviceArena::free_block(void* p) {
    for (size_t i = 0; i < blocks.size(); ++i)
        if (blocks[i] == p) {
            cudaFree(p);
            blocks.erase(blocks.begin() + (long)i);
            return;
        }
}
void DeviceArena::release() {
    for (void* b : blocks) cudaFree(b);
    blocks.clear();
}

cudaError_t ClipScratch::upload_vops(const ModeCtx& ctx, const LanePlan& plan, int frames, bool upload, const uint8_t** d_ops) {
    *d_ops = nullptr;
    if (!upload) return cudaSuccess;
    const size_t lanes = plan.op.size();
    vops.resize((size_t)frames * lanes);
    for (int t = 0; t < frames; ++t)
        for (size_t l = 0; l < lanes; ++l) {
            const uint8_t o = plan.op[l];
            vops[(size_t)t * lanes + l] = o == LANE_HOLD ? LANE_HOLD : (t == 0 ? o : (uint8_t)LANE_RUN);
        }
    *d_ops = d_vops;
    return cudaMemcpyAsync(d_vops, vops.data(), vops.size(), cudaMemcpyHostToDevice, ctx.stream);
}

mc_status ClipScratch::copy_last_tap(const ModeCtx& ctx, const LanePlan& plan, int frames, size_t lane_floats) const {
    if (!ctx.float_out) return MC_OK;
    const float* last = fout + (size_t)(frames - 1) * plan.op.size() * lane_floats;
    return for_each_run(plan.op.size(), [&](size_t l) { return plan.op[l] != LANE_HOLD; }, [&](size_t a, size_t b) -> mc_status {
        MCK(cudaMemcpyAsync(ctx.float_out + a * lane_floats, last + a * lane_floats, (b - a) * lane_floats * sizeof(float),
                            cudaMemcpyDeviceToDevice, ctx.stream));
        return MC_OK;
    });
}

void MotionMode::drop_groups() {
    for (Group& g : groups) {
        if (g.stream) { cudaStreamSynchronize(g.stream); cudaStreamDestroy(g.stream); }
        if (g.done) cudaEventDestroy(g.done);
    }
    groups.clear();
    if (ev_fork) { cudaEventDestroy(ev_fork); ev_fork = nullptr; }
}

void MotionMode::reset() {
    drop_groups();
    arena.release();
    clip.arena.release();
    clip = Clip{};
    lv.clear(); G.clear(); hi.clear(); lo.clear(); M.clear();
    lab16 = nullptr;
    d_coef = nullptr;
    coef_host.clear();
    coef_key.clear();
    lane_ema = nullptr; lane_chroma = lane_gain = nullptr;
    lab16_frame = false;
    gauss_frame = false;
    allocated = false;
    empty = true;
    ab_bounded = true;
}

// (Re)builds the lane groups — their streams, events and TMA descriptors — over the existing buffers; the temporal state
// is untouched, so the option can change between frames (profile_kernels forces one group).
mc_status MotionMode::make_groups(const ModeCtx& ctx) {
    // lane groups: automatic = two chains once each has >= 8 streams.  The stages contend for the same L1 data pipe,
    // so co-residency buys little beyond filling each other's tails.
    drop_groups();
    groups_req = ctx.opt.lane_groups;
    int ng = groups_req > 0 ? groups_req : std::min(2, lanes / 8);
    ng = std::max(1, std::min(ng, lanes));
    groups.assign((size_t)ng, Group{});
    for (int g = 0; g < ng; ++g) {
        Group& grp = groups[(size_t)g];
        grp.lane0 = (int)((long long)lanes * g / ng);
        grp.lanes = (int)((long long)lanes * (g + 1) / ng) - grp.lane0;
        if (ng > 1) {
            MCK(cudaStreamCreateWithFlags(&grp.stream, cudaStreamNonBlocking));
            MCK(cudaEventCreateWithFlags(&grp.done, cudaEventDisableTiming));
        }
        // TMA descriptors for the f32 inputs and the state planes of the fused level kernels, over this group's planes
        const size_t p0 = (size_t)grp.lane0 * channels;
        const int gp = grp.lanes * channels;
        grp.tmaps.assign((size_t)levels + 1, TensorMapStorage{});
        grp.tmaps_hi.assign((size_t)levels + 1, TensorMapStorage{});
        grp.tmaps_lo.assign((size_t)levels + 1, TensorMapStorage{});
        grp.tmap_valid.assign((size_t)levels + 1, 0);
        for (int l = 1; l < levels; ++l) {
            const Level& L = lv[(size_t)l];
            grp.tmap_valid[(size_t)l] = make_level_tensor_map(&grp.tmaps[(size_t)l], G[(size_t)l] + p0 * L.plane, L, gp) &&
                                        make_level_tensor_map(&grp.tmaps_hi[(size_t)l], hi[(size_t)l] + p0 * L.plane, L, gp, true) &&
                                        make_level_tensor_map(&grp.tmaps_lo[(size_t)l], lo[(size_t)l] + p0 * L.plane, L, gp, true) ? 1 : 0;
        }
    }
    if (ng > 1) MCK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    return MC_OK;
}

// TemporalFilter.cpp:11-12
static void ema_cutoffs(const mc_params& p, double& c_lo, double& c_hi) {
    c_lo = p.coLow == 0 ? 0.01 : p.coLow;
    c_hi = p.coHigh;
}
static bool cutoffs_in_01(double c_lo, double c_hi) { return c_lo >= 0 && c_lo <= 1 && c_hi >= 0 && c_hi <= 1; }   // NaN is not
// The parameters' part of the L-only condition (see luma_only): a zero chroma factor and bounded gains
static bool luma_params(const mc_params& p, const std::vector<float>& g) {
    if ((float)p.chromAttenuation * (1.0f / 64.0f) != 0.0f) return false;   // the egress's chroma64, as the device forms it
    for (float v : g)
        if (!(std::fabs(v) <= 0x1p64f)) return false;
    return true;
}

mc_status MotionMode::allocate(const ModeCtx& ctx, int width, int height, int nchannels, int nlevels) {
    reset();
    levels = nlevels; channels = nchannels; w = width; h = height;
    faithful = ctx.opt.faithful_level0;
    from_state = ctx.opt.band_from_state;
    const size_t planes = (size_t)lanes * channels;
    lv.resize((size_t)levels + 1);
    int cw = w, ch = h;
    for (int l = 0; l <= levels; ++l) {
        lv[(size_t)l] = make_level(cw, ch);
        cw = (cw + 1) / 2;
        ch = (ch + 1) / 2;
    }
    G.assign((size_t)levels + 1, nullptr);
    hi.assign((size_t)levels + 1, nullptr);
    lo.assign((size_t)levels + 1, nullptr);
    M.assign((size_t)levels + 1, nullptr);
    for (int l = 0; l <= levels; ++l) {
        const size_t n = planes * lv[(size_t)l].plane;
        const bool band_level = l < levels;                       // bands 0..levels-1, residual = levels
        const bool live = band_level && l >= 1;                   // bands whose gain can be non-zero
        if (l >= 1) MCK(arena.alloc(&G[(size_t)l], n));
        if (live || faithful) {
            MCK(arena.alloc(&hi[(size_t)l], n));
            MCK(arena.alloc(&lo[(size_t)l], n));
        }
        // M_l: the amplified band of level l, overwritten by the collapsed cur_l.  With band_from_state the bands are
        // rebuilt from hi/lo by their consumers and only cur_2 .. cur_{levels-2} are materialised.
        if (live && (!from_state || (l >= 2 && l <= levels - 2))) MCK(arena.alloc(&M[(size_t)l], n));
    }
    if (channels == 3) {
        pitch16 = round_up(w, 64);
        plane16 = (size_t)h * pitch16;
        void* p = nullptr;
        MCK(arena.alloc_bytes(&p, planes * plane16 * sizeof(int16_t)));
        lab16 = (int16_t*)p;
    }
    MCK_ST(make_groups(ctx));
    allocated = true;
    return MC_OK;
}

mc_status MotionMode::process(const ModeCtx& ctx, const FrameIO& io_in, const mc_params& p, int nlevels, int* produced, int frames) {
    *produced = 0;
    if (!allocated || faithful != ctx.opt.faithful_level0 || from_state != ctx.opt.band_from_state) {
        if (allocated) *ctx.held_lost = true;
        mc_status st = allocate(ctx, io_in.w, io_in.h, io_in.channels, nlevels);
        if (st != MC_OK) return st;
    } else if (groups_req != ctx.opt.lane_groups) {
        mc_status st = make_groups(ctx);
        if (st != MC_OK) return st;
    }
    // Per-lane ops: a lane without state takes its first frame (MagnifyCore.hpp:98-103) while the others run; a held lane is
    // skipped by every kernel.  Uniform frames pass no op array and `first` says which of the two paths all lanes take.
    plan.make(ctx.lane_ops, lanes, empty);
    if (plan.n_hold == lanes) {   // every lane held: nothing to do
        plan.produced(ctx, false, false, produced);
        return MC_OK;
    }
    const bool first = plan.n_first == lanes;  // MagnifyCore.hpp:98
    FrameIO io = io_in;
    MCK(plan.upload(ctx, &io.ops));
    motion_gains(p.amplification, p.coWavelength, levels, w, h, gains);
    double c_lo, c_hi;
    ema_cutoffs(p, c_lo, c_hi);
    bool in01 = cutoffs_in_01(c_lo, c_hi), luma_ok = luma_params(p, gains);
    MCK_ST(lane_table(ctx, &in01, &luma_ok));
    // a frame of a lane with state steps the EMAs (a clip's later frames always do)
    if ((plan.n_run > 0 || frames > 1) && !in01) ab_bounded = false;
    const bool luma = luma_ok && luma_only(ctx);

    lab16_frame = false;   // a clip converts into its own scratch; a frame call rewrites lab16 below
    gauss_frame = false;   // likewise its pyramid (clip.G)
    if (frames > 1) {
        MCK_ST(run_clip(ctx, io, p, frames, first, c_lo, c_hi, luma));
    } else if (groups.size() == 1) {
        MCK_ST(run_group(ctx, io, p, groups[0], first, c_lo, c_hi, luma));
    } else {
        // fork: every group's chain starts after whatever the caller queued on the handle's stream (the frame upload),
        // join: the handle's stream continues after all of them (the download / the caller's next use of `out`)
        MCK(cudaEventRecord(ev_fork, ctx.stream));
        for (Group& g : groups) {
            MCK(cudaStreamWaitEvent(g.stream, ev_fork, 0));
            ModeCtx gctx = ctx;
            gctx.stream = g.stream;
            const mc_status st = run_group(gctx, io, p, g, first, c_lo, c_hi, luma);
            if (st != MC_OK) return st;
            MCK(cudaEventRecord(g.done, g.stream));
            MCK(cudaStreamWaitEvent(ctx.stream, g.done, 0));
        }
    }
    empty = false;
    lab16_frame = frames == 1 && lab16;
    gauss_frame = frames == 1;
    // state-carry pass (analysis_only): the temporal state is up to date, only first frames are produced; a clip's later
    // frames run for the lanes that are not held
    plan.produced(ctx, !ctx.opt.analysis_only || first, true, produced, frames, !ctx.opt.analysis_only);
    return MC_OK;
}

// Lanes with parameters of their own (ctx.lane_params): builds the per-lane table and uploads it on the handle's stream
// when its contents changed (the kernels of earlier frames precede the copy in stream order).  ANDs every lane's
// cutoff and L-only conditions into *in01 / *luma_ok, which a shared decision needs to hold for every lane.
mc_status MotionMode::lane_table(const ModeCtx& ctx, bool* in01, bool* luma_ok) {
    lane_ema = nullptr; lane_chroma = lane_gain = nullptr;
    if (!ctx.lane_params) return MC_OK;
    const size_t n = (size_t)lanes, bytes = n * 4 * sizeof(double) + n * sizeof(float) + (size_t)(levels + 1) * n * sizeof(float);
    // The table follows from the lanes' six fields alone (levels, w and h are fixed until the next allocation, which
    // clears the key), so it is rebuilt and uploaded only when they change.
    bool same = d_coef && coef_key.size() == 6 * n;
    for (size_t k = 0; same && k < n; ++k) same = std::memcmp(&ctx.lane_params[k].amplification, &coef_key[6 * k], 6 * sizeof(double)) == 0;
    if (!same) {
        coef_key.resize(6 * n);
        coef_host.assign(bytes, 0);
        double* ema = reinterpret_cast<double*>(coef_host.data());
        float* chroma = reinterpret_cast<float*>(ema + 4 * n);
        float* gain = chroma + n;
        std::vector<float> g;
        coef_in01 = coef_luma = true;
        for (size_t k = 0; k < n; ++k) {
            const mc_params& q = ctx.lane_params[k];
            std::memcpy(&coef_key[6 * k], &q.amplification, 6 * sizeof(double));
            double c_lo, c_hi;
            ema_cutoffs(q, c_lo, c_hi);
            ema[4 * k] = c_hi; ema[4 * k + 1] = 1 - c_hi; ema[4 * k + 2] = c_lo; ema[4 * k + 3] = 1 - c_lo;
            chroma[k] = (float)q.chromAttenuation;
            motion_gains(q.amplification, q.coWavelength, levels, w, h, g);
            for (int l = 0; l <= levels; ++l) gain[(size_t)l * n + k] = g[(size_t)l];
            coef_in01 = coef_in01 && cutoffs_in_01(c_lo, c_hi);
            coef_luma = coef_luma && luma_params(q, g);
        }
        if (!d_coef) MCK(arena.alloc_bytes(&d_coef, bytes));
        // pageable source: staged before the call returns; stream-ordered after the kernels that read the old contents
        MCK(cudaMemcpyAsync(d_coef, coef_host.data(), bytes, cudaMemcpyHostToDevice, ctx.stream));
    }
    *in01 = *in01 && coef_in01;
    *luma_ok = *luma_ok && coef_luma;
    lane_ema = static_cast<const double*>(d_coef);
    lane_chroma = reinterpret_cast<const float*>(lane_ema + 4 * n);
    lane_gain = lane_chroma + n;
    return MC_OK;
}

// ---- the launch set around the level kernels, shared by run_group (io: one group's lanes) and run_clip (io: every
// frame's lanes) ----

// production path, >= 2 levels: one fused kernel converts u8 BGR to Lab16 planes and also builds G1; otherwise the
// level-0 kernel builds G1 (from the Lab16 planes, or from gray frames directly)
bool MotionMode::fused_ingest() const { return channels == 3 && !faithful && levels >= 2; }
// the first level the level loop runs: level 0 only builds G1 unless the faithful option is on
int MotionMode::first_level() const { return fused_ingest() ? 1 : ((levels >= 2 || faithful) ? 0 : levels); }

mc_status MotionMode::ingest(const ModeCtx& ctx, const FrameIO& io, int16_t* lab, float* g1) {
    if (fused_ingest()) LAUNCH("ingest_lab", 0, launch_ingest_lab(io, *ctx.tables, lab, pitch16, plane16, g1, lv[1], ctx.stream));
    else if (channels == 3) LAUNCH("lab16", 0, launch_lab16(io, *ctx.tables, lab, pitch16, plane16, ctx.stream));
    return MC_OK;
}

// The level kernel's arguments that do not depend on the path: level l reads g[l] (level 0: the Lab16 planes or the
// gray frames) and writes g[l + 1], from plane p0 on; the state planes hi / lo likewise.
LevelArgs MotionMode::level_args(int l, const std::vector<float*>& g, size_t p0, const int16_t* lab, const FrameIO& io, bool first,
                                 double c_lo, double c_hi) const {
    LevelArgs a;
    if (l == 0) {
        if (channels == 3) {
            a.in_kind = 1; a.g = lab; a.in_plane = plane16; a.in_row = pitch16;
            a.sc[0] = 100.0f / 16384.0f; a.of[0] = 0.0f;
            a.sc[1] = a.sc[2] = 1.0f / 64.0f; a.of[1] = a.of[2] = -128.0f;
        } else {
            a.in_kind = 2; a.g = io.in; a.in_plane = io.in_lane_stride; a.in_row = (int)io.in_step;
            a.sc[0] = 0.003921568859368563f;
        }
    } else {
        a.in_kind = 0; a.g = g[(size_t)l] + p0 * lv[(size_t)l].plane; a.in_plane = lv[(size_t)l].plane; a.in_row = lv[(size_t)l].pitch;
    }
    auto off = [&](float* base, int k) { return base ? base + p0 * lv[(size_t)k].plane : nullptr; };
    a.channels = channels;
    a.lf = lv[(size_t)l]; a.lc = lv[(size_t)l + 1];
    a.g_next = off(g[(size_t)l + 1], l + 1);
    a.hi = off(hi[(size_t)l], l); a.lo = off(lo[(size_t)l], l);
    a.first = first ? 1 : 0;
    a.band = (l >= 1 || faithful) ? 1 : 0;
    a.c_hi = c_hi; a.one_minus_c_hi = 1 - c_hi; a.c_lo = c_lo; a.one_minus_c_lo = 1 - c_lo;
    a.gain = gains[(size_t)l];
    const size_t lane0 = p0 / (size_t)channels;
    a.lane_ema = lane_ema ? lane_ema + 4 * lane0 : nullptr;
    a.lane_gain = gain_of(l, (int)lane0);
    return a;
}

// faithful_level0: st.lowpassHi/Lo[levels] = the residual g_res of a lane's first frame (MagnifyCore.hpp:100-101), for the
// lanes [lane0, lane0 + n) that take it; one copy pair per run of such lanes.
mc_status MotionMode::copy_residual(const ModeCtx& ctx, const float* g_res, int lane0, int n) {
    if (!faithful) return MC_OK;
    const size_t lane_floats = (size_t)channels * lv[(size_t)levels].plane;
    return for_each_run((size_t)n, [&](size_t i) { return plan.op[(size_t)lane0 + i] == LANE_FIRST; }, [&](size_t a, size_t b) -> mc_status {
        const size_t o = ((size_t)lane0 + a) * lane_floats, len = (b - a) * lane_floats;
        LAUNCH("copy", levels, launch_copy_planes(hi[(size_t)levels] + o, g_res + o, len, ctx.stream));
        LAUNCH("copy", levels, launch_copy_planes(lo[(size_t)levels] + o, g_res + o, len, ctx.stream));
        return MC_OK;
    });
}

// analysis_only (state-carry pass): lanes on their first frame are still converted (no motion), running lanes produce
// nothing.
mc_status MotionMode::egress_first_frames(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, float* fout,
                                          bool first) {
    if (first || plan.n_first > 0) MCK_ST(egress(ctx, io, p, lane0, lab, BandSrc{}, BandSrc{}, fout, !first, false));
    return MC_OK;
}

// The egress launch over io's lanes, the first of them the handle's lane lane0 (a clip's virtual lane v is lane v % lanes)
mc_status MotionMode::egress(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, const BandSrc& m1,
                             const BandSrc& c2, float* fout, bool first_only, bool luma) {
    LAUNCH("egress", 0, launch_egress(io, *ctx.tables, lab, pitch16, plane16, m1, lv[levels >= 1 ? 1 : 0], c2, lv[levels >= 2 ? 2 : 0],
                                      (float)p.chromAttenuation, fout, ctx.stream, ctx.opt.egress_strip, first_only, luma,
                                      lane_chroma ? lane_chroma + lane0 : nullptr, std::min(io.lanes, lanes)));
    return MC_OK;
}

// L-only synthesis (DESIGN §4).  The egress adds chroma/64 * u to a and b, u being the a / b motion; when that factor is
// zero and u is finite the sum is a, b bit for bit, so only the L planes need to be synthesised.  u is finite when every
// gain is finite with |g| <= 2^64 and the a / b state is bounded: EMAs with cutoffs in [0, 1] are convex combinations of
// bands (|band| <= 256), so |m_l| <= 512 * 2^64 and the collapse sums stay far below FLT_MAX.  The strip egress alone has
// an L-only form; the tile egress always synthesises every channel.  The parameters' part (luma_params) is checked by the
// caller, for every lane.
bool MotionMode::luma_only(const ModeCtx& ctx) const { return channels == 3 && ctx.opt.egress_strip && ab_bounded; }

// Synthesis: residual and finest band are zero (MagnifyCore.hpp:130-131), so the collapse starts from band levels-1
// (cur_{levels-1} = 0 + m_{levels-1}) and writes cur_l to out(l) down to level 2; levels 1 and 0 are folded into egress.
// band(l) is where level l's amplified band is found.  Without motion (first frames) egress converts the input as it is.
// luma: L-only synthesis, the collapses run over each lane's L plane only.
template <class Band, class Out>
mc_status MotionMode::synthesize(const ModeCtx& ctx, const FrameIO& io, const mc_params& p, int lane0, const int16_t* lab, float* fout, bool motion,
                                 bool luma, Band band, Out out) {
    BandSrc m1, c2;
    if (motion && levels >= 2) {
        auto cur = [&](int l) { return l == levels - 1 ? band(l) : BandSrc{out(l), nullptr, 1.0f}; };
        const int planes = luma ? io.lanes : io.lanes * channels, stride = luma ? channels : 1;
        for (int l = levels - 2; l >= 2; --l)
            LAUNCH("collapse", l, launch_collapse(lv[(size_t)l], lv[(size_t)l + 1], band(l), cur(l + 1), out(l), planes,
                                                  ctx.stream, io.ops, channels, stride));
        m1 = band(1);
        if (levels >= 3) c2 = cur(2);
    }
    return egress(ctx, io, p, lane0, lab, m1, c2, fout, false, luma);
}

// One group's launch set for one frame: lanes [g.lane0, g.lane0 + g.lanes) on ctx.stream.
mc_status MotionMode::run_group(const ModeCtx& ctx, const FrameIO& io_all, const mc_params& p, Group& g, bool first, double c_lo, double c_hi,
                                bool luma) {
    FrameIO io = io_all;
    io.in = io_all.in + (size_t)g.lane0 * io_all.in_lane_stride;
    io.out = io_all.out + (size_t)g.lane0 * io_all.out_lane_stride;
    io.lanes = g.lanes;
    if (io.ops) io.ops += g.lane0;   // the op array is indexed by the handle's lane
    const size_t p0 = (size_t)g.lane0 * channels;
    auto off = [&](float* base, int l) { return base ? base + p0 * lv[(size_t)l].plane : nullptr; };
    int16_t* lab = lab16 ? lab16 + p0 * plane16 : nullptr;
    float* fout = ctx.float_out ? ctx.float_out + (size_t)g.lane0 * w * h * channels : nullptr;

    MCK_ST(ingest(ctx, io, lab, off(G[1], 1)));
    for (int l = first_level(); l < levels; ++l) {
        LevelArgs a = level_args(l, G, p0, lab, io, first, c_lo, c_hi);
        if (l >= 1 && g.tmap_valid[(size_t)l] && ctx.opt.use_tma) {
            a.tmap = &g.tmaps[(size_t)l];
            a.tmap_hi = &g.tmaps_hi[(size_t)l];
            a.tmap_lo = &g.tmaps_lo[(size_t)l];
        }
        a.m = (first || from_state) ? nullptr : off(M[(size_t)l], l);
        a.m_luma = luma;
        a.planes = g.lanes * channels;
        a.ops = io.ops;
        if (a.band) LAUNCH("level", l, launch_level(a, ctx.stream));
        else LAUNCH("down", l, launch_down(a, ctx.stream));
    }
    MCK_ST(copy_residual(ctx, G[(size_t)levels], g.lane0, g.lanes));
    if (ctx.opt.analysis_only) return egress_first_frames(ctx, io, p, g.lane0, lab, fout, first);
    auto band = [&](int l) {
        return from_state ? BandSrc{off(hi[(size_t)l], l), off(lo[(size_t)l], l), gains[(size_t)l], gain_of(l, g.lane0)}
                          : BandSrc{off(M[(size_t)l], l), nullptr, 1.0f};
    };
    return synthesize(ctx, io, p, g.lane0, lab, fout, !first, luma, band, [&](int l) { return off(M[(size_t)l], l); });
}

// One clip: the launch set of run_group over V = frames * lanes virtual lanes, with the level kernels replaced by
// k_level_clip (state in registers across the clip).  Synthesis reads the stored bands M_l; a lane's first frame has
// M = +-0 there, which gives the first-frame output without a branch.  Lane groups do not apply: one chain.
mc_status MotionMode::run_clip(const ModeCtx& ctx, const FrameIO& io0, const mc_params& p, int frames, bool first, double c_lo, double c_hi,
                               bool luma) {
    const int vl = frames * lanes;
    MCK_ST(ClipScratch::grow(clip, ctx, vl, channels == 3 ? (size_t)vl * channels * plane16 * sizeof(int16_t) : 0, (size_t)w * h * channels,
                             [&]() -> mc_status {
        const size_t vplanes = (size_t)vl * channels;
        clip.G.assign((size_t)levels + 1, nullptr);
        clip.M.assign((size_t)levels + 1, nullptr);
        clip.tmaps.assign((size_t)levels + 1, TensorMapStorage{});
        clip.tmap_valid.assign((size_t)levels + 1, 0);
        for (int l = 1; l <= levels; ++l) {
            MCK(clip.arena.alloc(&clip.G[(size_t)l], vplanes * lv[(size_t)l].plane));
            if (l < levels) MCK(clip.arena.alloc(&clip.M[(size_t)l], vplanes * lv[(size_t)l].plane));
            if (l < levels) clip.tmap_valid[(size_t)l] = make_level_tensor_map(&clip.tmaps[(size_t)l], clip.G[(size_t)l], lv[(size_t)l], (int)vplanes) ? 1 : 0;
        }
        return MC_OK;
    }));
    FrameIO io = io0;   // every frame of every lane
    io.lanes = vl;
    MCK(clip.upload_vops(ctx, plan, frames, plan.mixed(), &io.ops));

    MCK_ST(ingest(ctx, io, clip.lab16, clip.G[1]));
    for (int l = first_level(); l < levels; ++l) {
        LevelArgs a = level_args(l, clip.G, 0, clip.lab16, io, first, c_lo, c_hi);
        if (l >= 1 && clip.tmap_valid[(size_t)l] && ctx.opt.use_tma) a.tmap = &clip.tmaps[(size_t)l];
        a.m = ctx.opt.analysis_only ? nullptr : clip.M[(size_t)l];
        a.m_luma = luma;
        if (a.band) {
            a.planes = lanes * channels; a.ops = io0.ops;   // state planes, per-lane ops of the clip's first frame
            LAUNCH("level_clip", l, launch_level_clip(a, frames, ctx.stream));
        } else {
            a.planes = vl * channels; a.ops = io.ops;
            LAUNCH("down", l, launch_down(a, ctx.stream));
        }
    }
    MCK_ST(copy_residual(ctx, clip.G[(size_t)levels], 0, lanes));   // frame 0 is the first `lanes` virtual lanes
    // state-carry pass: only the clip's first frame can produce; it is frame 0's egress of a frame call, so the float
    // tap is written in place
    if (ctx.opt.analysis_only) return egress_first_frames(ctx, io0, p, 0, clip.lab16, ctx.float_out, first);
    MCK_ST(synthesize(ctx, io, p, 0, clip.lab16, ctx.float_out ? clip.fout : nullptr, true, luma,
                      [&](int l) { return BandSrc{clip.M[(size_t)l], nullptr, 1.0f}; }, [&](int l) { return clip.M[(size_t)l]; }));
    return clip.copy_last_tap(ctx, plan, frames, (size_t)w * h * channels);
}

void MotionMode::find_state(const char* name, int level, StateRef& out) {
    out = StateRef{};
    if (!std::strcmp(name, "lab16")) {
        if (level == 0) lab16_state(lab16, lab16_frame, w, h, pitch16, plane16, out);
        return;
    }
    if (!allocated || empty || level < 0 || level > levels) return;
    if (!std::strcmp(name, "gauss")) {
        // read-only tap of G_1 .. G_levels of the last frame call (include/magcore_b200.h, at mc_get_state); with one
        // level and no faithful level 0 no kernel writes G_1 (the level loop is empty, the ingest is k_lab16)
        if (!gauss_frame || level < 1 || first_level() >= levels) return;
        const Level& l = lv[(size_t)level];
        out.ptr = G[(size_t)level]; out.rows = l.h; out.cols = l.w; out.channels = channels; out.pitch = l.pitch;
        out.plane_stride = l.plane; out.read_only = true;
        return;
    }
    float* p = nullptr;
    if (!std::strcmp(name, "lowpassHi")) p = hi[(size_t)level];
    else if (!std::strcmp(name, "lowpassLo")) p = lo[(size_t)level];
    else if (!std::strcmp(name, "band")) p = M[(size_t)level];
    if (!p) return;
    const Level& l = lv[(size_t)level];
    out.ptr = p; out.rows = l.h; out.cols = l.w; out.channels = channels; out.pitch = l.pitch; out.plane_stride = l.plane;
}

void MotionMode::lane_planes(int lane, std::vector<LanePlane>& out) const {
    out.clear();
    if (!allocated) return;
    for (int l = 0; l <= levels; ++l) {
        const Level& L = lv[(size_t)l];
        for (float* p : {hi[(size_t)l], lo[(size_t)l]})
            if (p)   // a lane's channels are consecutive planes of h rows `pitch` apart: one block of channels * h rows
                out.push_back(LanePlane{p + (size_t)lane * channels * L.plane, (size_t)L.pitch * sizeof(float), (size_t)L.w * sizeof(float),
                                        (size_t)channels * L.h});
    }
}

}  // namespace mc
