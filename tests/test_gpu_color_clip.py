"""Color clips: mc_process_clip runs a Color clip as one launch set, the per-frame kernels over every frame of the clip at
once and the window filter frame by frame on the handle's ring.  T consecutive frames in one call must equal, bit for
bit, the same frames fed one frame call at a time: u8 outputs (the sentinel where a frame did not produce), produced
flags, mc_lane_produced, the float tap, and the read-only taps "gauss", "window", "filtered" and "up" afterwards, which
are those of the clip's last frame."""
import os

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_clip import check_clip, clip_frames, run_clip, run_frames
from test_gpu_lanes import COLOR_UI, proc

EMU = os.environ.get("MC_EMU") == "1"
TAPS = ("gauss", "window", "filtered", "up")
LIFECYCLE = (("color_lane_lifecycle", 1),)


def color_cfg(levels=2, fps=8.0, mode=O.MODE_COLOR):
    return make_cfgs(mode, *COLOR_UI[:5], levels, fps)[0]


def taps(p):
    """{(name, level): array} of every tap the handle serves (window / filtered: one level per column)"""
    out = {}
    for n in TAPS:
        for lvl in range(66):
            if p.state_dims(n, lvl)[0]:
                out[(n, lvl)] = p.get_state(n, lvl)
    return out


def assert_taps_equal(a, b, where=None, held=()):
    """every tap of `a` equals `b`'s; the "gauss" planes of `held` lanes are left out (they convert whatever the lane's
    input slot holds, which in a chain call with a front stage is staging the front skipped)"""
    ta, tb = taps(a), taps(b)
    assert sorted(ta) == sorted(tb), (where, sorted(set(ta) ^ set(tb)))
    keep = [k for k in range(next(iter(tb.values())).shape[0]) if k not in held] if tb else []
    for k in tb:
        x, y = (ta[k][keep], tb[k][keep]) if k[0] == "gauss" else (ta[k], tb[k])
        assert np.array_equal(x, y), (where, k)
    return tb


def check_color(w, h, c, steps, lanes=1, options=(), levels=2, fps=8.0, float_out=False):
    """Two handles with the same options take the same frames and events: `steps` is a list of
        ("clip", n)  a clip of n frames on the first handle, n frame calls on the second,
        ("frames", n)  n frame calls on both,   ("none", n)  a clip / n frame calls in mode None,
        ("fps", f) / ("levels", l) / ("size", (w, h))  from here on,   ("reset",)  mc_reset,
        ("restart", k) / ("hold", k, on)  a lane event on both;
    after every frame step the flags, the u8 outputs, mc_lane_produced, every tap and (float_out) the float tap are
    equal.  -> the first handle's flags per frame step."""
    opts = tuple(options) + ((("keep_float_output", 1),) if float_out else ())
    a, b = proc(lanes, opts), proc(lanes, opts)
    t, got = 0, []
    for i, step in enumerate(steps):
        kind = step[0]
        if kind == "fps":
            fps = step[1]
        elif kind == "levels":
            levels = step[1]
        elif kind == "size":
            w, h = step[1]
        elif kind == "reset":
            a.reset()
            b.reset()
        elif kind == "restart":
            a.restart_lane(step[1])
            b.restart_lane(step[1])
        elif kind == "hold":
            a.hold_lane(step[1], step[2])
            b.hold_lane(step[1], step[2])
        else:
            n = step[1]
            cfg = color_cfg(levels, fps, O.MODE_NONE if kind == "none" else O.MODE_COLOR)
            fr = clip_frames(t, n, lanes, w, h, c)
            fa, oa = run_clip(a, fr, cfg) if kind in ("clip", "none") else run_frames(a, fr, cfg)
            fb, ob = run_frames(b, fr, cfg)
            assert np.array_equal(fa, fb), (i, fa.tolist(), fb.tolist())
            assert np.array_equal(oa, ob), i
            assert np.array_equal(a.lane_produced(), b.lane_produced()), i
            assert_taps_equal(a, b, i)
            if float_out:
                assert np.array_equal(a.float_output(w, h, c), b.float_output(w, h, c)), i
            got.append(fa)
            t += n
    a.close()
    b.close()
    return got


SIZES = [(96, 64), (91, 67)]   # 91 x 67: the pyrUp chain ends at 92 x 68, so the bilinear resize runs

# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("w,h", SIZES)
def test_warmup_inside_a_clip_crosses_two_columns_and_the_cap(w, h, c):
    """8 fps: a window of at most 16 columns.  The first clip holds frames that pass through and the first filtered
    ones, the second crosses the cap."""
    got = check_color(w, h, c, [("clip", 5), ("clip", 14), ("clip", 3)])
    assert got[0][:, 0].tolist() == [0, 1, 1, 1, 1] and got[1].all() and got[2].all()


@pytest.mark.parametrize("c", [3, 1])
def test_clip_longer_than_the_window(c):
    """40 and 37 frames against a 16-slot window: slots are overwritten twice within one clip"""
    check_color(91, 67, c, [("clip", 40), ("clip", 37)], float_out=True)


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("levels", [1, 2, 3, 4])
@pytest.mark.parametrize("w,h", SIZES + [(33, 41)])
def test_levels_and_sizes(w, h, levels, c):
    check_color(w, h, c, [("clip", 3), ("clip", 6)], levels=levels)


def test_framerate_changes_between_clips():
    """8 -> 30 fps grows the ring and lays the full, wrapped window out in order; 30 -> 8 keeps a longer window; 7 fps
    lowers the cap again; each change is taken at a clip's first frame"""
    check_color(91, 67, 3, [("clip", 20), ("fps", 30.0), ("clip", 10), ("fps", 8.0), ("clip", 6), ("frames", 2),
                            ("fps", 7.0), ("clip", 9), ("fps", 30.0), ("clip", 4)], float_out=True)


def test_interleaves_with_frame_calls_reset_size_change_and_mode_none():
    check_color(96, 64, 3, [("frames", 3), ("clip", 4), ("frames", 2), ("clip", 5), ("reset",), ("clip", 3),
                            ("size", (91, 67)), ("clip", 4), ("none", 2), ("clip", 3), ("levels", 3), ("clip", 2),
                            ("frames", 1)])


def test_existing_clip_checker():
    """the checker the other modes' clips pass (check_lanes_clip compares state planes, which Color has none of: the lane
    cases below compare every lane's taps instead)"""
    check_clip(O.MODE_COLOR, COLOR_UI, 120, 90, 3, [("clip", 4), ("frames", 2), ("clip", 5), ("size", (97, 61)), ("clip", 3)])


@pytest.mark.parametrize("c", [3, 1])
def test_lanes_restart_hold_and_different_window_lengths(c):
    """3 lanes with their own windows: restarts and holds at clip starts give lanes of different lengths (one transform
    per lane), held lanes keep their bytes and float tap; a frame-rate change while a lane is held"""
    steps = [("clip", 6), ("restart", 1), ("hold", 2, 1), ("clip", 5), ("hold", 2, 0), ("clip", 7), ("restart", 0),
             ("clip", 12), ("hold", 1, 1), ("fps", 30.0), ("clip", 4), ("hold", 1, 0), ("clip", 3), ("frames", 2),
             ("restart", 0), ("restart", 1), ("restart", 2), ("clip", 3)]
    check_color(91, 67, c, steps, lanes=3, options=LIFECYCLE, float_out=True)


def test_every_lane_held():
    got = check_color(96, 64, 3, [("clip", 3), ("hold", 0, 1), ("hold", 1, 1), ("clip", 2), ("hold", 0, 0), ("clip", 2)],
                      lanes=2, options=LIFECYCLE)
    assert not got[1].any() and got[2][:, 0].all() and not got[2][:, 1].any()


def test_refusal_without_the_option_leaves_the_state_unchanged():
    """a hold or a single-lane restart of a multi-lane handle without color_lane_lifecycle: MC_ERR_UNSUPPORTED before
    anything runs; taps and window are those before the call, and the handle continues like its twin"""
    cfg = color_cfg()
    w, h, c, lanes = 96, 64, 3, 2
    a, b = proc(lanes), proc(lanes)
    fr = clip_frames(0, 6, lanes, w, h, c)
    run_clip(a, fr, cfg)
    run_frames(b, fr, cfg)
    before = assert_taps_equal(a, b)
    for event, undo in (("hold", lambda: a.hold_lane(1, False)), ("restart", None)):
        a.hold_lane(1) if event == "hold" else a.restart_lane(1)
        with pytest.raises(L.MagcoreError) as e:
            run_clip(a, clip_frames(6, 3, lanes, w, h, c), cfg)
        assert e.value.status == capi.MC_ERR_UNSUPPORTED
        got = taps(a)
        assert sorted(got) == sorted(before) and all(np.array_equal(got[k], before[k]) for k in before)
        if undo:
            undo()
    a.reset()   # the pending restart is dropped with the state
    b.reset()
    fr = clip_frames(6, 4, lanes, w, h, c)
    fa, oa = run_clip(a, fr, cfg)
    fb, ob = run_frames(b, fr, cfg)
    assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
    assert_taps_equal(a, b)
    a.close()
    b.close()


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
def test_1080p():
    check_color(1920, 1080, 3, [("clip", 8), ("clip", 8)], levels=3, fps=30.0, float_out=True)


# ---- the chain, compose and 4:2:2 calls with frames > 1 against their frame loops -------------------------------------

def split_calls(call, n, lanes, src):
    """call(src_slice, frames) -> tuple of [frames, lanes] flags and [V]-major arrays; -> the frame loop's, stacked"""
    parts = [call(src[t * lanes:(t + 1) * lanes], 1) for t in range(n)]
    return tuple(None if p[0] is None else np.concatenate(p) for p in zip(*parts))


def check_chain_calls(kind, w, h, steps, lanes=2, settings=None):
    """Handle A takes `kind` calls of n frames, handle B the same frames one call each; flags, lane flags, every output
    buffer and every tap are equal after each step ("clip", n), ("restart", k), ("hold", k, on)."""
    from test_gpu_chain_lanes import chain_cfg, device_call
    from test_gpu_compose import Canvas, compose_call, sources
    from test_gpu_nv12 import Layout
    from test_gpu_yuv422 import Yuv, from_bgr, yuv_device_call
    cfg = chain_cfg(O.MODE_COLOR, COLOR_UI, **(settings or {}))
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    for ch in (a, b):
        ch.magnifier.set_option("color_lane_lifecycle", 1)
    t, held = 0, set()
    for step in steps:
        if step[0] in ("restart", "hold"):
            for ch in (a, b):
                ch.magnifier.restart_lane(step[1]) if step[0] == "restart" else ch.magnifier.hold_lane(step[1], step[2])
            if step[0] == "hold":
                (held.add if step[2] else held.discard)(step[1])
            continue
        n = step[1]
        if kind == "chain":
            src, _ = sources(t, n, lanes, w, h, "bgr")

            def call(ch):
                return lambda s, f: (lambda r: (r[0], r[2], r[3]))(device_call(ch, cfg, s, f, w, h, 3))
        elif kind == "compose_nv12":
            src, _ = sources(t, n, lanes, w, h, "nv12")
            nv = Layout(w, h, pitch=w + 2, uv_row=h + 2)

            def call(ch):
                def run(s, f):
                    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, capi.MC_SPLIT_LEFT_RIGHT)
                    cv = Canvas(capi.MC_CANVAS_NV12, cw, chh, len(s), pad=4)
                    flags, _ = compose_call(ch.magnifier, cfg, s, f, w, h, 3, capi.MC_SPLIT_LEFT_RIGHT, cv.struct(), nv)
                    return flags, cv.dev.numpy(), None
                return run
        else:
            frames, _ = sources(t, n, lanes, w, h, "bgr")
            src = np.stack([from_bgr(f, capi.MC_YUV422_YUYV) for f in frames])
            lay = Yuv(w, h, capi.MC_YUV422_YUYV, pitch=2 * w + 4)

            def call(ch):
                return lambda s, f: (lambda r: (r[0], r[2], r[3]))(yuv_device_call(ch, cfg, s, f, lay))
        t += n
        ra = call(a)(src, n)
        rb = split_calls(call(b), n, lanes, src)
        for x, y in zip(ra, rb):
            assert (x is None and y is None) or np.array_equal(x, y), step
        assert np.array_equal(a.magnifier.lane_produced(), b.magnifier.lane_produced()), step
        assert_taps_equal(a.magnifier, b.magnifier, step, held)


CHAIN_STEPS = [("clip", 3), ("clip", 4), ("restart", 1), ("hold", 0, 1), ("clip", 3), ("hold", 0, 0), ("clip", 2)]


@pytest.mark.parametrize("settings", [dict(), dict(down=2, gray=True)], ids=["no_front", "front"])
def test_chain_device_clip_equals_its_frame_loop(settings):
    check_chain_calls("chain", 96, 64, CHAIN_STEPS, settings=settings)


def test_chain_compose_nv12_clip_equals_its_frame_loop():
    check_chain_calls("compose_nv12", 96, 64, CHAIN_STEPS, settings=dict(down=2))


def test_chain_yuv422_clip_equals_its_frame_loop():
    check_chain_calls("yuv422", 96, 64, CHAIN_STEPS)


# ---- launches ----------------------------------------------------------------------------------------------------------

def check_launches(w=91, h=67, levels=2, c=3):
    """On a handle with a full window a clip of T frames launches 2 * levels + 6 kernels (+1 for the resize) once and
    the append, the two transforms and the mask once per frame, under their frame-call names; a warm-up frame that
    filters nothing only appends.  Profiling does not change the bytes."""
    cfg = color_cfg(levels)
    sw, sh = w, h
    for _ in range(levels):
        sw, sh = (sw + 1) // 2, (sh + 1) // 2
    resize = 1 if (sw << levels, sh << levels) != (w, h) else 0   # the pyrUp chain misses the frame size
    once = 2 * levels + 6 + resize
    p, q = proc(1, (("profile_kernels", 1),)), proc(1)
    fr = clip_frames(0, 3, 1, w, h, c)
    n0 = p.launch_count
    run_clip(p, fr, cfg)
    run_clip(q, fr, cfg)
    assert p.launch_count - n0 == once + 3 + 3 * 2    # frame 0 appends only
    prof = p.profile_read()
    assert prof[("ring_append", 0)][0] == 3 and prof[("cufft_r2c", 0)][0] == 2
    t = 3
    for n in (2, 17, 8):
        fr = clip_frames(t, n, 1, w, h, c)
        n0 = p.launch_count
        fa, oa = run_clip(p, fr, cfg)
        fb, ob = run_clip(q, fr, cfg)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
        assert p.launch_count - n0 == once + 4 * n, n
        prof = {k: v[0] for k, v in p.profile_read().items()}
        want = {("u8_to_planes", 0): 1, ("minmax_window", 0): 1, ("select", 0): 1, ("minmax_out", 0): 1,
                ("color_egress", 0): 1, ("ring_append", 0): n, ("cufft_r2c", 0): n, ("mask_mul", 0): n, ("cufft_c2r", 0): n}
        want.update({("gauss_down", lvl): 1 for lvl in range(levels)})
        want.update({("pyrup2x", lvl): 1 for lvl in range(levels)})
        if resize:
            want[("resize", 0)] = 1
        assert prof == want, (n, prof)
        t += n
    p.close()
    q.close()


def test_launch_count_and_profile_names():
    check_launches()
    check_launches(96, 64, 3, 1)
