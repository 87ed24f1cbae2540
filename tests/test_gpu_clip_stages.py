"""Clips (mc_process_clip) stage by stage: the clip-only kernels k_level_clip (Laplace), k_riesz_phase_clip (Phase) and
Color's batched k_minmax / k_select / reconstruction over V = frames * lanes virtual lanes, tied to the host references
of the stage suites (tests/test_gpu_laplace_stages.py, test_gpu_phase_stages.py, test_gpu_color_stages.py).

The method is a reference twin.  A twin handle with the same options takes the clip's frames as frame calls, and every
one of those frame calls goes through its mode's stage checker (`check_frame`), which compares each kernel with a
float64 or bit-exact host reference of its own operation.  After every clip the clip handle must equal the twin bit for
bit: the u8 output of every frame (the sentinel where a frame did not produce), the produced flags and
mc_lane_produced, every state plane, the float tap, and in Color every read-only tap (the clip's last frame's).  So a
clip is checked against the references on exactly the content and geometry it ran.

Where a clip's result can be computed without the twin it is also checked directly:
  Laplace  the state after the clip == T iterations of ema_exact from the state set with mc_set_state (values of both
           signs up to about 1e7), each frame's band read from a handle that takes that frame as its first frame (its
           hi is the band); the faithful residual of a lane on its first frame == G_levels of the clip's frame 0
  Color    check_frame on the clip handle itself: its taps are those of the clip's last frame (gauss, window, filtered,
           up, the float tap) and the u8 output of that frame; the extremum of the last frame's window in the last
           virtual lane lands where it was put, and the output stretch's extremes in tail columns and the last row
  Limit    a clip of exactly frames * lanes = MC_MAX_LANES virtual lanes equals its twin, and one more is refused with
           the state and the output buffer untouched.

Lane lifecycle in a clip: restarts and holds are taken at the clip's first frame.  A held lane is skipped for the whole
clip; a restarted lane takes frame 0 as its first frame and runs from frame 1 on."""
import collections
import ctypes as C
import os

import numpy as np
import pytest

from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
import test_gpu_color_stages as CS
import test_gpu_laplace_stages as LS
import test_gpu_phase_stages as PS

pytestmark = pytest.mark.gpu
F32 = np.float32
EMU = os.environ.get("MC_EMU") == "1"
SENTINEL = 0xA5
U8P = C.POINTER(C.c_uint8)


# ---- calls with sentinel-filled output buffers -------------------------------------------------------------------------
def _rows(frames, pad):
    """[..., lanes, h, w, c] u8 -> [..., lanes, h, w * c + pad] rows (pad bytes 0xEE)"""
    *lead, h, w, c = frames.shape
    buf = np.full((*lead, h, w * c + pad), 0xEE, np.uint8)
    buf[..., : w * c] = frames.reshape(*lead, h, w * c)
    return buf


def frame_call(p, frames, prm, pad=0):
    """mc_process of [lanes][h][w][c] -> (lane flags u8 [lanes], out [lanes][h][w * c + pad])"""
    lanes, h, w, c = frames.shape
    buf = _rows(frames, pad)
    out = np.full_like(buf, SENTINEL)
    p.process_host(buf.ctypes.data, w, h, c, buf.shape[-1], prm, out.ctypes.data, buf.shape[-1])
    return p.lane_produced().astype(np.uint8), out


def clip_call(p, frames, prm, pad=0, status=capi.MC_OK):
    """mc_process_clip of [T][lanes][h][w][c] -> (flags u8 [T][lanes], out [T][lanes][h][w * c + pad])"""
    T, lanes, h, w, c = frames.shape
    buf = _rows(frames, pad)
    out = np.full_like(buf, SENTINEL)
    flags = np.zeros((T, lanes), np.uint8)
    st = p._lib.mc_process_clip(p._h, buf.ctypes.data, T, w, h, c, buf.shape[-1], C.byref(prm), out.ctypes.data,
                                buf.shape[-1], flags.ctypes.data_as(U8P))
    assert st == status, (st, status)
    return flags, out


def planes_of(p, names, levels):
    return {(n, l): p.get_state(n, l) for n in names for l in range(levels + 1) if p.state_dims(n, l)[0] > 0}


def assert_twin(kp, rp, flags, out, rflags, rout, names, levels, w, h, c, ctx, fout=True, lost=()):
    """The clip handle kp after a clip (flags, out) == the twin rp after the same frames as frame calls; the state planes
    of the lanes in `lost` (state the handle dropped: they restart on release) are not compared"""
    assert np.array_equal(flags, rflags), (ctx, flags.tolist(), rflags.tolist())
    for t in range(len(out)):
        assert np.array_equal(out[t], rout[t]), (ctx, "u8", t)
    assert np.array_equal(kp.lane_produced(), rp.lane_produced()), ctx
    a, b = planes_of(kp, names, levels), planes_of(rp, names, levels)
    assert a.keys() == b.keys(), (ctx, sorted(a), sorted(b))
    keep = [k for k in range(kp.lanes) if k not in lost]
    for key in a:
        assert np.array_equal(a[key][keep], b[key][keep], equal_nan=True), (ctx, "state", key)
    if fout:
        assert np.array_equal(kp.float_output(w, h, c), rp.float_output(w, h, c), equal_nan=True), (ctx, "float tap")


def apply_events(handles, evs, first, held):
    for e in evs:
        for hd in handles:
            if e[0] == "restart":
                hd.p.restart_lane(e[1])
            elif e[0] == "hold":
                hd.p.hold_lane(e[1], e[2])
        if e[0] == "restart":
            first[e[1]] = True
        elif e[0] == "hold":
            held[e[1]] = bool(e[2])


# ---- Laplace ---------------------------------------------------------------------------------------------------------------
LAPLACE_STATE = ("lowpassHi", "lowpassLo")


def run_laplace_clips(w, h, c=3, lanes=1, levels=4, clips=(3, 2), kind="noise", chroma=50, options=(), pad=0,
                      events=None, set_state=(), co_low=None, co_high=None, seed=0):
    """Clips of clips[i] frames on one handle; a twin takes the same frames as frame calls, each checked stage by stage
    (LS.check_frame), and the clip handle equals it after every clip.  The state after each clip also equals the EMA
    chain of ema_exact over the clip's bands from the state before it.  events[i]: [("restart", k) | ("hold", k, on)]
    before clip i; set_state: clip indices before which every state plane of both handles is replaced by the same
    random values of both signs up to about 1e7."""
    rng = np.random.default_rng(seed)
    lv = LS.eff_levels(w, h, levels)
    opts = dict(options)
    faithful, from_state = opts.get("faithful_level0", 0) == 1, opts.get("band_from_state", 1) == 1
    analysis_only = opts.get("analysis_only", 0) == 1
    kh, rh, tw = LS.Handle(lanes, options), LS.Handle(lanes, options), LS.Handle(lanes, options)
    stats = collections.Counter()
    prm_p = LS.params(levels, chroma=chroma, co_low=co_low, co_high=co_high)
    gains = LS.gains_of(prm_p, lv, w, h)
    c_hi, c_lo = prm_p.coHigh, prm_p.coLow if prm_p.coLow != 0 else 0.01
    first, held = [True] * lanes, [False] * lanes
    ab_bounded, state_set, t0 = True, False, 0
    for i, T in enumerate(clips):
        apply_events((kh, rh), (events or {}).get(i, []), first, held)
        if i in set_state:
            state_set = True
            for l in range(lv + 1):
                if kh.p.state_dims("lowpassHi", l)[0] > 0:
                    for nm in LAPLACE_STATE:
                        a = kh.tap(nm, l)
                        v = (rng.standard_normal(a.shape) * 10.0 ** rng.integers(-3, 7, a.shape)).astype(F32)
                        kh.p.set_state(nm, l, v)
                        rh.p.set_state(nm, l, v)
        ops0 = ["hold" if held[k] else "first" if first[k] else "run" for k in range(lanes)]
        before = planes_of(kh.p, LAPLACE_STATE, lv)
        frames = np.stack([LS.frames_of(kind, t0 + t, lanes, w, h, c) for t in range(T)])
        rflags, rout, bands = [], [], []
        for t in range(T):
            ops = ["hold" if held[k] else "first" if first[k] else "run" for k in range(lanes)]
            if "run" in ops and not (0 <= c_lo <= 1 and 0 <= c_hi <= 1):
                ab_bounded = False
            luma = (c == 3 and opts.get("egress_strip", 1) == 1 and ab_bounded and F32(chroma) * LS.INV64 == 0
                    and all(abs(g) <= 2.0 ** 64 for g in gains))
            prev = {"gauss": {l: rh.tap("gauss", l) for l in range(1, lv + 1)},
                    "hi": {l: rh.tap("lowpassHi", l) for l in range(lv + 1)},
                    "lo": {l: rh.tap("lowpassLo", l) for l in range(lv + 1)},
                    "band": {l: rh.tap("band", l) for l in range(lv + 1)}}
            fl, out = frame_call(rh.p, frames[t], prm_p, pad)
            rflags.append(fl)
            rout.append(out)
            tw.p.reset()
            tw.frame(frames[t], prm_p, pad=pad)
            bands.append({l: tw.tap("lowpassHi", l) for l in range(lv + 1) if tw.p.state_dims("lowpassHi", l)[0] > 0})
            if not analysis_only:   # the checker's egress expects synthesis
                prm = dict(lv=lv, faithful=faithful, from_state=from_state, co_high=c_hi, co_low=prm_p.coLow, gains=gains,
                           luma=luma, chroma=prm_p.chromAttenuation, state_set=state_set)
                LS.check_frame(rh, tw, frames[t], out, ops, prev, prm, stats, (w, h, c, lanes, i, t))
            for k in range(lanes):
                first[k] = first[k] and held[k]
        flags, out = clip_call(kh.p, frames, prm_p, pad)
        assert_twin(kh.p, rh.p, flags, out, np.stack(rflags), rout, LAPLACE_STATE, lv, w, h, c, (w, h, c, lanes, i),
                    fout=not analysis_only)
        # directly: T iterations of the EMA from the state before the clip
        after = planes_of(kh.p, LAPLACE_STATE, lv)
        for (nm, l), got in after.items():
            cc = c_hi if nm == "lowpassHi" else c_lo
            for k in range(lanes):
                if ops0[k] == "hold":
                    assert np.array_equal(got[k], before[nm, l][k]), (i, nm, l, k)
                    continue
                if l == lv and faithful:   # the residual: G_levels of the lane's first frame, else untouched
                    want = bands[0][l][k] if ops0[k] == "first" else before[nm, l][k]
                    assert np.array_equal(got[k], want), (i, nm, l, k)
                    continue
                s, ts = (bands[0][l][k], range(1, T)) if ops0[k] == "first" else (before[nm, l][k], range(T))
                for t in ts:
                    s = LS.ema_exact(s, bands[t][l][k], 1 - cc, cc)
                bad = got[k] != s
                assert not bad.any(), (i, "ema chain", nm, l, k, int(bad.sum()), np.argwhere(bad)[:4].tolist())
        t0 += T
    for hd in (kh, rh, tw):
        hd.close()
    for key in ("B", "B'"):
        LS.SEEN[key] = max(LS.SEEN[key], stats[key])
    return stats


# The Laplace seam sweep (LS.SWEEP: strip seams, level tiles, every width residue mod 4, padded rows, gray and colour,
# lanes and lane groups, levels smaller than one tile) with two clips each.  The clip lengths cover T in {1, 2, 3, 4, 5,
# 8, 17}, in both positions: with TMA buffer t & 1's barrier is waited on with parity (t >> 1) & 1, so bar[0] returns to
# a phase from T >= 5 (t = 0, 2, 4) and bar[1] from T >= 6 (t = 1, 3, 5); T = 8 and 17 reuse both phases of both.
CLIP_TS = (1, 2, 3, 4, 5, 8, 17)
LAPLACE_CASES = [(*case, (CLIP_TS[i % 7], CLIP_TS[(i + 3) % 7])) for i, case in enumerate(LS.SWEEP)]


@pytest.mark.parametrize("w,h,c,lanes,levels,options,pad,kind,clips", LAPLACE_CASES)
@pytest.mark.parametrize("chroma", [50, 0])
def test_laplace_clip_on_the_seam_sweep(w, h, c, lanes, levels, options, pad, kind, clips, chroma):
    if EMU and w * h * max(clips) > 257 * 129 * 5:
        clips = tuple(min(T, 5) for T in clips)   # the large sizes' longest clips are too slow for the CPU emulation
    run_laplace_clips(w, h, c, lanes, levels, clips=clips, kind=kind, chroma=chroma, options=options, pad=pad,
                      seed=w * 1000 + h)


def interior_level_tiles(w, h, l=1):
    """k_level_clip's interior tiles at level l of a w x h frame: x0 >= 4, x0 + TW + 4 <= wf, y0 >= 4, y0 + TH + 3 <= hf
    with TW x TH = 64 x 32 (mc_laplace.cu); they take the staged window as loaded, without the reflect patch"""
    wf, hf = (w + 2 ** l - 1) >> l, (h + 2 ** l - 1) >> l
    return sum(1 for x0 in range(0, wf, 64) for y0 in range(0, hf, 32)
               if x0 >= 4 and x0 + 68 <= wf and y0 >= 4 and y0 + 35 <= hf)


@pytest.mark.parametrize("T", CLIP_TS)
@pytest.mark.parametrize("tma", [1, 0])
def test_laplace_clip_ema_chain_from_set_state(T, tma):
    """State of both signs up to about 1e7 set before each clip; coLow 0 (the driver takes 0.01) with coHigh above 1,
    then ordinary cutoffs.  133 x 70 has border level-1 tiles only (level 1 is 67 x 35).  400 x 300 (level 1 200 x 150)
    has interior level-1 tiles, the tiles a large frame spends its time in; at 266 x 134 level 1 is 133 x 67, exactly
    the size where the tile at (64, 32) becomes interior, and 264 x 132 (132 x 66) is one row short of it."""
    assert interior_level_tiles(133, 70) == 0 and interior_level_tiles(264, 132) == 0
    assert interior_level_tiles(400, 300) > 0 and interior_level_tiles(266, 134) == 1
    for c in (3, 1):
        run_laplace_clips(133, 70, c, 1, 4, clips=(2, T), set_state=(1,), co_low=0.0, co_high=1.5,
                          options=(("use_tma", tma),), seed=T)
    run_laplace_clips(133, 70, 3, 2, 4, clips=(1, T), set_state=(0, 1), co_low=0.3, co_high=0.9,
                      options=(("use_tma", tma),), seed=T + 100)
    Ti = min(T, 5) if EMU else T   # the large frames' longest clips are too slow for the CPU emulation
    run_laplace_clips(400, 300, 3, 1, 4, clips=(2, Ti), set_state=(1,), co_low=0.0, co_high=1.5,
                      options=(("use_tma", tma),), seed=T + 200)
    for w, h, c in ((266, 134, 1), (264, 132, 3)):
        run_laplace_clips(w, h, c, 2, 4, clips=(1, Ti), set_state=(0, 1), co_low=0.3, co_high=0.9,
                          options=(("use_tma", tma),), seed=T + w)


@pytest.mark.parametrize("options", [(("faithful_level0", 1),), (("faithful_level0", 1), ("use_tma", 0)),
                                     (("band_from_state", 0),), (("lane_groups", 2),)])
@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_options(options, c):
    """faithful_level0: level 0 runs k_level_clip<IN_LAB16> (colour) / <IN_U8> (gray) and the residual is kept;
    band_from_state 0; lane_groups 2 on an uneven split (5 lanes: 2 + 3) — a clip runs one chain"""
    lanes = 5 if dict(options).get("lane_groups") else 2
    run_laplace_clips(71, 37, c, lanes, 4, clips=(3, 4, 2), kind="shadows", options=options, pad=1,
                      set_state=(1,), seed=c)


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_lanes_run_first_and_hold(c):
    """3 lanes: before clip 1 lane 1 restarted (FIRST at the clip's frame 0 while lane 0 runs) and lane 2 held for the
    whole clip; released before clip 2.  Also with faithful level 0 and state set before the mixed clip."""
    events = {1: [("restart", 1), ("hold", 2, 1)], 2: [("hold", 2, 0)]}
    for opts in ((), (("faithful_level0", 1), ("use_tma", 0))):
        run_laplace_clips(135, 66, c, 3, 4, clips=(2, 5, 3), events=events, options=opts, set_state=(1,), seed=7)


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_analysis_only(c):
    """Only the handle's first frame is produced; the state moves as in frame calls"""
    events = {1: [("restart", 1)]}
    run_laplace_clips(83, 45, c, 2, 4, clips=(4, 3), events=events, options=(("analysis_only", 1),), set_state=(1,))


# ---- Phase -----------------------------------------------------------------------------------------------------------------
def run_phase_clips(w, h, lanes=1, levels=8, clips=(3, 2), kind="synth", alpha=50, wavelength=50.0, lo=0.4, hi=3.0,
                    fps=30.0, options=(), events=None, seed=0, egress_frames=None):
    """Clips of clips[i] frames; a twin takes the same frames as frame calls, each checked stage by stage
    (PS.check_frame), and the clip handle equals it after every clip.  events[i]: [("restart", k) | ("hold", k, on) |
    ("cutoffs", lo, hi)] before clip i; egress_frames: the twin's frames after this many skip the egress's cv2
    comparison.  -> branch counters of the twin's frames"""
    rng = np.random.default_rng(seed)
    lv = PS.eff_levels(w, h, levels)
    assert lv >= 2
    kh, rh = PS.Handle(lanes, options), PS.Handle(lanes, options)
    stats = collections.Counter()
    stats["amp_ref_err"] = 0.0
    first, held = [True] * lanes, [False] * lanes
    analysis_only = dict(options).get("analysis_only", 0) == 1
    t0, lost = 0, set()
    for i, T in enumerate(clips):
        evs = (events or {}).get(i, [])
        apply_events((kh, rh), evs, first, held)
        lost = {k for k in lost if held[k]}
        changed = False
        for e in evs:
            if e[0] == "cutoffs":
                changed = changed or (lo, hi) != e[1:]
                lo, hi = e[1:]
        cfg, ocfg = make_cfgs(O.MODE_PHASE, alpha, wavelength, lo, hi, 0, levels, fps)
        prm_p = _to_mc(cfg)
        frames = np.stack([PS.content(kind, t0 + t, lanes, w, h, rng) for t in range(T)])
        rflags, rout = [], []
        for t in range(T):
            ops = ["hold" if held[k] else "first" if first[k] else "run" for k in range(lanes)]
            rebuild = changed and "run" in ops
            changed = changed and not rebuild
            before = rh.states(lv) if t0 + t > 0 else None
            prev = rh.taps(lv)
            fl, out = frame_call(rh.p, frames[t], prm_p)
            rflags.append(fl)
            rout.append(out)
            if rebuild and "hold" in ops:
                # new cutoffs zero every lane's registers: a held lane loses its state and restarts on release
                after = rh.states(lv)
                for k in range(lanes):
                    if ops[k] == "hold":
                        first[k] = True
                        lost.add(k)
                        for key in before:
                            before[key][k] = after[key][k]
            prm = dict(alpha=alpha, coWavelength=ocfg.magnification.coWavelength, lo=lo, hi=hi, fps=fps,
                       analysis_only=analysis_only, egress_cv2=egress_frames is None or t0 + t < egress_frames)
            PS.check_frame(rh, frames[t], out.reshape(lanes, h, w, 3), ops, before, prev, lv, prm, rebuild, stats)
            for k in range(lanes):
                first[k] = first[k] and held[k]
        flags, out = clip_call(kh.p, frames, prm_p)
        assert_twin(kh.p, rh.p, flags, out, np.stack(rflags), rout, PS.STATE, lv, w, h, 3, (w, h, lanes, i),
                    fout=not analysis_only, lost=lost)
        t0 += T
    kh.close()
    rh.close()
    return stats


# The Phase seam sweep (PS.SWEEP: every width residue mod 8 at level 0, border-only and interior 32 x 16 phase tiles)
PHASE_CASES = [(w, h, lanes, tma, (CLIP_TS[i % 7], CLIP_TS[(i + 2) % 7])) for i, (w, h, lanes, tma) in enumerate(PS.SWEEP_CASES)]


@pytest.mark.parametrize("w,h,lanes,tma,clips", PHASE_CASES)
def test_phase_clip_on_the_seam_sweep(w, h, lanes, tma, clips):
    """Clips of 1 .. 17 frames: the first clip holds the passthrough first frame.  Where the last multiple of 8 below a
    level's width is not a multiple of the 32-column tile (13, 31, 63, 67, 70, 139, ... at level 0), filter2D's scalar
    tail columns sit inside a tile whose x0 is below them"""
    if EMU:
        clips = tuple(min(T, 5) for T in clips)
    run_phase_clips(w, h, lanes, clips=(1,) + clips, options=(("use_tma", tma),), seed=w * 1000 + h)


@pytest.mark.parametrize("kind", PS.KINDS)
@pytest.mark.parametrize("tma", [0, 1])
def test_phase_clip_on_black_impulse_and_saturated_content(kind, tma):
    """192 x 128, 5 levels: the NaN patch of the phase kernel and, next to the windowbox, its clamp branch run inside a
    clip; clips of 2, 5 and 8 frames after the first.  On saturated content past the stage suite's three frames the
    frame path's egress is 8.3e-6 from cv2 on an H100, beyond the checker's 8e-6: there that one cv2 comparison is
    waived (the clip still equals the twin bit for bit, and the twin's u8 output still equals convertTo of its float
    tap)."""
    s = run_phase_clips(192, 128, 1, clips=(3, 2, 5, 8), kind=kind, options=(("use_tma", tma),),
                        egress_frames=3 if kind == "saturated" else None)
    if kind in ("blackrect", "windowbox"):
        assert s["nan_patch"] > 0 and s["amp_nan"] > 0 and s["nan_L"] > 0, s
    if kind == "windowbox":
        assert s["clamp"] > 0, s


@pytest.mark.parametrize("tma", [0, 1])
def test_phase_clip_cutoff_change_at_a_clip_start(tma):
    """New cutoffs at a clip's start rebuild the prior from that clip's frame 0 (rebuild_old: t == 0 only; frames 1.. of
    the clip take the previous frame); one lane restarted and one held across the change.  New cutoffs zero every lane's
    filter registers, so the held lane restarts when it is released a clip later: its planes are compared from then on
    (while it is held, frame calls leave a stale prior in them and a clip leaves them as they were)."""
    events = {1: [("cutoffs", 0.8, 3.0)], 2: [("cutoffs", 0.8, 2.0), ("restart", 1), ("hold", 2, 1)],
              3: [("hold", 2, 0)], 4: [("cutoffs", 0.5, 2.5)]}
    run_phase_clips(135, 40, 3, levels=4, clips=(3, 4, 3, 4, 3), events=events, kind="windowbox",
                    options=(("use_tma", tma),))


def test_phase_clip_lanes_run_first_and_hold():
    """3 lanes: lane 1 restarted (FIRST at frame 0 of the clip while lane 0 runs), lane 2 held for the whole clip; then
    a clip of FIRST + HOLD lanes only; then all run"""
    events = {1: [("restart", 1), ("hold", 2, 1)], 2: [("hold", 0, 1), ("restart", 1)], 3: [("hold", 0, 0), ("hold", 2, 0)]}
    run_phase_clips(135, 40, 3, levels=4, clips=(2, 4, 1, 3), kind="blackrect", events=events)


def test_phase_clip_analysis_only():
    """No frame is produced and the Riesz pair and amplitude are not written; the state moves as in frame calls"""
    run_phase_clips(96, 48, 2, levels=3, clips=(3, 4), options=(("analysis_only", 1),), events={1: [("restart", 0)]})


# ---- Color -----------------------------------------------------------------------------------------------------------------
def color_taps(hd, lv):
    """every read-only tap of a Color handle"""
    taps = {("gauss", l): hd.tap("gauss", l) for l in range(lv + 2)}
    taps.update({("up", l): hd.tap("up", l) for l in range(lv + 3)})
    for nm in ("window", "filtered"):
        taps.update({(nm, j): hd.tap(nm, j) for j in range(hd.columns(nm))})
    return taps


def assert_taps_equal(a, b, ctx):
    assert a.keys() == b.keys(), ctx
    for key in a:
        assert (a[key] is None) == (b[key] is None) and (a[key] is None or np.array_equal(a[key], b[key])), (ctx, key)


def run_color_clips(w, h, c, lanes, clips, levels=2, fps=8.0, lo=0.5, hi=4.0, alpha=100, pad=0, events=None,
                    frames_of=None, seed=0, options=()):
    """Clips of clips[i] frames (fps of clip i: fps or fps[i]); a twin takes the same frames as frame calls, each
    produced one in lock-step checked stage by stage (CS.check_frame), and the clip handle equals it after every clip in
    outputs, flags, lane flags, every tap and the float tap; the clip handle's own taps are also checked stage by stage
    (they are its last frame's).  frames_of(t) -> [lanes][h][w][c].  -> (clip handle, its last flags and out)"""
    rng = np.random.default_rng(seed)
    lv = CS.eff_levels(w, h, levels)
    kh, rh = CS.Handle(lanes, options), CS.Handle(lanes, options)
    held, restarted = [False] * lanes, [True] * lanes
    lockstep, t0 = True, 0   # every lane's window has the same length: the checker's filter reference applies
    for i, T in enumerate(clips):
        f_i = fps[i] if isinstance(fps, (tuple, list)) else fps
        cfg = make_cfgs(O.MODE_COLOR, alpha, 0.0, lo, hi, 0, levels, f_i)[0]
        prm_p = _to_mc(cfg)
        evs = (events or {}).get(i, [])
        apply_events((kh, rh), evs, restarted, held)
        lockstep = lockstep and not evs
        frames = np.stack([frames_of(t0 + t) if frames_of else CS.noise_frames(rng, lanes, h, w, c) for t in range(T)])
        rflags, rout = [], []
        for t in range(T):
            fl, out = frame_call(rh.p, frames[t], prm_p, pad)
            rflags.append(fl)
            rout.append(out)
            o = out[..., : w * c].reshape(lanes, h, w, c)
            if lockstep and fl.all() and rh.columns("filtered") == rh.columns("window") >= 2:
                CS.check_frame(rh, frames[t], o, lv, alpha, lo, hi, f_i)
        flags, out = clip_call(kh.p, frames, prm_p, pad)
        assert_twin(kh.p, rh.p, flags, out, np.stack(rflags), rout, (), lv, w, h, c, (w, h, c, lanes, i))
        assert_taps_equal(color_taps(kh, lv), color_taps(rh, lv), i)
        o = out[-1][..., : w * c].reshape(lanes, h, w, c)
        if lockstep and flags[-1].all() and kh.columns("filtered") == kh.columns("window") >= 2:
            CS.check_frame(kh, frames[-1], o, lv, alpha, lo, hi, f_i)   # the clip handle's own taps: its last frame
        t0 += T
    rh.close()
    return kh, flags, out, frames


@pytest.mark.parametrize("w,h,c,lanes", CS.SWEEP[::2])
def test_color_clip_on_the_seam_sweep(w, h, c, lanes):
    """Deepest pyramid the size allows, padded rows: a clip through the warm-up (frame 0 does not produce), then clips
    of 2 and 5 frames"""
    kh, *_ = run_color_clips(w, h, c, lanes, (3, 2, 5), levels=8, pad=5, seed=w * 1000 + h)
    kh.close()


def test_color_clip_window_wraps_inside_a_clip_and_framerate_changes_at_clip_starts():
    """8 fps (a 16-column window): a clip of 10, then one of 12 that wraps the window inside it; 30 fps (grows to 64
    while full) at a clip's start; back to 8 fps (the longer window keeps its length); 7 fps"""
    for c, lanes in ((3, 1), (1, 3)):
        kh, *_ = run_color_clips(91, 67, c, lanes, (10, 12, 6, 5, 4), fps=(8.0, 8.0, 30.0, 8.0, 7.0), lo=0.8, hi=1.2)
        kh.close()


def test_color_clip_lanes_restart_and_hold():
    """3 lanes: a restart in warm-up, a hold across the wrap, a restart after it (the lifecycle option)"""
    events = {1: [("restart", 1)], 2: [("hold", 2, 1)], 4: [("hold", 2, 0)], 5: [("restart", 0)]}
    kh, *_ = run_color_clips(91, 67, 3, 3, (4, 5, 9, 3, 4, 6), lo=0.8, hi=1.2, events=events, options=CS.LIFECYCLE)
    kh.close()


def flicker_clip(w, h, c, lanes, levels, n, lane, ch, y, x, slot, sign):
    """CS.flicker_case as one clip of n frames: the filtered window of the clip's last frame in `lane` (the last virtual
    lane when lane = lanes - 1) has its maximum (sign +1) or minimum (-1) exactly at (slot, ch, y, x); the clip equals
    its twin and its last frame's taps pass the stage checker"""
    lv = CS.eff_levels(w, h, levels)
    assert lv == levels
    fps, lo, hi = 8.0, 0.8, 1.2
    resp = CS.filter64(np.eye(n), lo, hi, fps)[0][:, 0]
    t0 = (slot - int(np.argmax(resp))) % n
    base = np.random.default_rng(7).integers(96, 160, size=(lanes, h, w, c))
    r = 1 << (levels - 1)
    sh, sw = (h + (1 << levels) - 1) >> levels, (w + (1 << levels) - 1) >> levels

    def bump(f, k, cy, cx, cc, a):
        f[k, max(cy * 2 * r - r, 0):cy * 2 * r + r + 1, max(cx * 2 * r - r, 0):cx * 2 * r + r + 1, cc] += a

    def frame(t):
        f = base.copy()
        if t == t0:
            for k in range(lanes):
                if k == lane:
                    bump(f, k, y, x, ch, 90 * sign)
                else:
                    bump(f, k, sh // 2, sw // 2, 0, 40 * sign)
        return np.clip(f, 0, 255).astype(np.uint8)

    kh, flags, out, frames = run_color_clips(w, h, c, lanes, (n,), levels=levels, lo=lo, hi=hi, frames_of=frame)
    assert flags[1:].all()
    filt = np.stack([kh.tap("filtered", k) for k in range(kh.columns("filtered"))], axis=1)
    assert filt.shape[1:] == (n, c, sh, sw)
    at = np.unravel_index(np.argmax(sign * filt[lane]), filt[lane].shape)
    assert at == (slot, ch, y, x), (at, (slot, ch, y, x))
    kh.close()


@pytest.mark.parametrize("sign", [1, -1])
@pytest.mark.parametrize("w,h,c,lanes,levels", CS.GEOMS)
def test_color_clip_extremum_in_the_last_element_of_the_last_virtual_lane(w, h, c, lanes, levels, sign):
    """CS.GEOMS: both sides of k_minmax's vector / scalar path, one and several CTAs a virtual lane, padded lanes"""
    sh, sw = (h + 1) // 2, (w + 1) // 2
    flicker_clip(w, h, c, lanes, levels, 7, lanes - 1, c - 1, sh - 1, sw - 1, 6, sign)


@pytest.mark.parametrize("w,h,c,lanes,levels", CS.GEOMS[:2] + CS.GEOMS[4:])
def test_color_clip_extremum_in_the_first_element_first_slot(w, h, c, lanes, levels):
    flicker_clip(w, h, c, lanes, levels, 5, lanes - 1, 0, 0, 0, 0, -1)


@pytest.mark.skipif(EMU, reason="70 lanes are too slow for the CPU emulation")
@pytest.mark.parametrize("w,h", [(64, 48), (128, 96)])
def test_color_clip_extremum_in_the_last_of_280_virtual_lanes(w, h):
    """70 lanes x 4 frames: k_minmax's grid is capped at 592 / 280 + 1 = 3 CTAs a virtual lane, so at 128 x 96 (9216
    floats a lane) each thread strides"""
    flicker_clip(w, h, 3, 70, 1, 4, 69, 2, h // 2 - 1, w // 2 - 1, 3, 1)


def stretch_clip(w, h, c, lanes, lane, lo_at, hi_at):
    """CS.stretch_case as one 2-frame clip: amplification 0, so the clip's last frame is the contrast stretch of its input;
    the extremes 3 and 250 of `lane` at lo_at / hi_at ((y, x, channel))"""
    frames = np.full((lanes, h, w, c), 128, np.uint8)
    frames[:, h // 2, w // 2, 0], frames[:, h // 2, w // 2 + 1, 0] = 40, 200
    frames[lane][lo_at], frames[lane][hi_at] = 3, 250

    def frame(t):
        f = frames.copy()
        f[:, 0, w // 2, 0] = 100 + 20 * t
        return f

    kh, flags, out, clip = run_color_clips(w, h, c, lanes, (2,), levels=1, lo=0.8, hi=1.2, alpha=0, frames_of=frame)
    assert flags.tolist() == [[0] * lanes, [1] * lanes]
    o = out[1][..., : w * c].reshape(lanes, h, w, c)
    assert np.array_equal(o[lane], CS.stretch_exact(clip[1][lane].astype(F32)))
    assert o[lane].min() == 0 and o[lane].max() == 255
    kh.close()


@pytest.mark.parametrize("w", [12, 13, 14, 15, 7])
@pytest.mark.parametrize("c", [1, 3])
def test_color_clip_stretch_extremes_in_the_tail_columns_and_last_row(w, c):
    h = 9
    for x in range(4 * (w >> 2), w):
        stretch_clip(w, h, c, 1, 0, (h - 1, x, c - 1), (h - 2, x, 0))
    stretch_clip(w, h, c, 1, 0, (h - 1, w - 1, c - 1), (0, 0, 0))
    stretch_clip(w, h, c, 3, 2, (0, 0, 0), (h - 1, w - 1, c - 1))   # the last of 6 virtual lanes


# ---- the virtual-lane limit ------------------------------------------------------------------------------------------------
LIMIT = [(1, capi.MC_MAX_LANES), (64, capi.MC_MAX_LANES // 64)]


def limit_case(mode, c, lanes, T):
    """One clip of exactly T * lanes = MC_MAX_LANES virtual lanes of 24 x 16 frames (12288 planes in grid.z for colour)
    == a twin that takes the same frames as T frame calls, bit for bit; then a clip of one more virtual lane is refused
    and leaves the state, every Color tap, the float tap and the output buffer as they were"""
    assert T * lanes == capi.MC_MAX_LANES
    w, h = 24, 16
    ui = {O.MODE_LAPLACE: (20, 50.0, 0.4, 3.0, 50, 4), O.MODE_PHASE: (50, 50.0, 0.4, 3.0, 0, 3),
          O.MODE_COLOR: (100, 0.0, 0.8, 1.2, 0, 2)}[mode]
    names = {O.MODE_LAPLACE: LAPLACE_STATE, O.MODE_PHASE: PS.STATE, O.MODE_COLOR: ()}[mode]
    prm_p = _to_mc(make_cfgs(mode, *ui)[0])
    kh, rh = CS.Handle(lanes), CS.Handle(lanes)
    rng = np.random.default_rng(lanes + c)
    # a smooth picture per lane that moves a little every frame, with noise on top
    yy, xx = np.mgrid[0:h, 0:w]
    frames = np.empty((T, lanes, h, w, c), np.uint8)
    for t in range(T):
        for k in range(lanes):
            base = 128 + 60 * np.sin((xx + 0.7 * t + 3 * k) / 5.0) * np.cos((yy - 0.3 * t) / 4.0)
            frames[t, k] = np.clip(base[..., None] + rng.integers(-8, 9, (h, w, c)), 0, 255).astype(np.uint8)
    rflags, rout = [], []
    for t in range(T):
        fl, out = frame_call(rh.p, frames[t], prm_p)
        rflags.append(fl)
        rout.append(out)
    flags, out = clip_call(kh.p, frames, prm_p)
    lv = 8
    assert flags[1:].all()
    assert_twin(kh.p, rh.p, flags, out, np.stack(rflags), rout, names, lv, w, h, c, (mode, c, lanes))
    if mode == O.MODE_COLOR:
        assert_taps_equal(color_taps(kh, lv), color_taps(rh, lv), "limit")
    # one virtual lane too many: refused, nothing changes
    kept = planes_of(kh.p, names, lv)
    kept_taps = color_taps(kh, lv) if mode == O.MODE_COLOR else {}
    fout = kh.p.float_output(w, h, c)
    big = np.concatenate([frames, frames[:1]])   # one more frame: MC_MAX_LANES + lanes virtual lanes
    fl, o = clip_call(kh.p, big, prm_p, status=capi.MC_ERR_INVALID)
    assert (o == SENTINEL).all() and not fl.any()
    after = planes_of(kh.p, names, lv)
    assert after.keys() == kept.keys()
    for key in kept:
        assert np.array_equal(after[key], kept[key], equal_nan=True), key
    assert np.array_equal(kh.p.float_output(w, h, c), fout, equal_nan=True)
    assert_taps_equal(color_taps(kh, lv) if mode == O.MODE_COLOR else {}, kept_taps, "refused")
    # and the handle goes on as its twin does
    nxt = frames[:2]
    flags, out = clip_call(kh.p, nxt, prm_p)
    rflags, rout = zip(*(frame_call(rh.p, f, prm_p) for f in nxt))
    assert_twin(kh.p, rh.p, flags, out, np.stack(rflags), rout, names, lv, w, h, c, (mode, c, lanes, "after"))
    if mode == O.MODE_COLOR:
        assert_taps_equal(color_taps(kh, lv), color_taps(rh, lv), "after")
    kh.close()
    rh.close()


@pytest.mark.skipif(EMU, reason="4096 virtual lanes are too slow for the CPU emulation")
@pytest.mark.parametrize("lanes,T", LIMIT)
@pytest.mark.parametrize("mode,c", [(O.MODE_LAPLACE, 3), (O.MODE_LAPLACE, 1), (O.MODE_PHASE, 3), (O.MODE_COLOR, 3),
                                    (O.MODE_COLOR, 1)])
def test_clip_at_exactly_max_lanes_virtual_lanes(mode, c, lanes, T):
    limit_case(mode, c, lanes, T)
