"""Color lanes with their own windows (option "color_lane_lifecycle"): every lane of a multi-lane Color handle must behave,
bit for bit, like its own 1-lane handle fed that lane's frames — its window restarted where the lane is restarted, not
fed at all while the lane is held, and each window following the frame rate under the rule of a 1-lane handle.  The
outputs are the witness: Color keeps its window internal."""
import ctypes as C
import os

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O
from common import make_cfgs, u8_diff
from test_gpu_lanes import COLOR_UI, SENTINEL, lane_frame, proc, process_raw, stack

LIFECYCLE = (("color_lane_lifecycle", 1),)
EMU = os.environ.get("MC_EMU") == "1"


def color_cfg(fps, ui=COLOR_UI):
    return make_cfgs(O.MODE_COLOR, *ui, fps)[0]


def apply(p, events):
    for e in events:
        if e[0] == "hold":
            p.hold_lane(e[1], e[2])
        else:
            p.restart_lane(e[1])


def run_lanes(w, h, c, lanes, n, events, fps=lambda t: 8.0, ui=COLOR_UI):
    """A `lanes`-lane handle takes n frame calls, events[t] ([("restart", k) | ("hold", k, on)]) applied before frame t.
    -> [(produced, out, flags)] per frame."""
    m = proc(lanes, LIFECYCLE)
    got = []
    for t in range(n):
        apply(m, events.get(t, []))
        got.append(process_raw(m, stack(t, lanes, w, h, c), color_cfg(fps(t), ui)))
    m.close()
    return got


def references(w, h, c, lanes, n, events, fps=lambda t: 8.0, ui=COLOR_UI):
    """Lane k's 1-lane handle (the option set) fed lane k's frames, restarted where lane k is, skipped while it is held
    -> per lane, per frame: None (held) or (produced, out)."""
    refs = [proc(1, LIFECYCLE) for _ in range(lanes)]
    held = [False] * lanes
    want = [[] for _ in range(lanes)]
    for t in range(n):
        for e in events.get(t, []):
            if e[0] == "hold":
                held[e[1]] = bool(e[2])
            else:
                refs[e[1]].restart_lane(0)
        cfg = color_cfg(fps(t), ui)
        for k in range(lanes):
            if held[k]:
                want[k].append(None)
                continue
            sprod, sout, _ = process_raw(refs[k], lane_frame(t, k, w, h, c)[None], cfg)
            want[k].append((sprod, sout[0]))
    for r in refs:
        r.close()
    return want


def assert_lanes_equal(got, want):
    """Flags and bytes of every lane and frame: a lane that did not produce keeps the sentinel."""
    for k, per_t in enumerate(want):
        for t, ref in enumerate(per_t):
            _, out, flags = got[t]
            if ref is None or not ref[0]:
                assert not flags[k] and (out[k] == SENTINEL).all(), (k, t)
            else:
                assert flags[k] and np.array_equal(out[k], ref[1]), (k, t, int(u8_diff(out[k], ref[1]).max()))
    assert all(g[0] == bool(g[2].any()) for g in got)


def check_lanes(w, h, c, lanes, n, events, fps=lambda t: 8.0, ui=COLOR_UI):
    got = run_lanes(w, h, c, lanes, n, events, fps, ui)
    assert_lanes_equal(got, references(w, h, c, lanes, n, events, fps, ui))
    return got


# ---- the scripts, shared with the emulation suite (tests/test_emu_color_lanes.py) ----------------------------------------
# 8 fps: window cap 16.  Restarts during warm-up (t 5) and after the window wrapped (t 25, 30)
RESTARTS = {5: [("restart", 1)], 25: [("restart", 2)], 30: [("restart", 1)]}
# holds spanning warm-up (lane 0, t 3..7) and the wrap (lane 2, t 14..21), two lanes held at once (t 31..33)
HOLDS = {3: [("hold", 0, 1)], 8: [("hold", 0, 0)], 14: [("hold", 2, 1)], 22: [("hold", 2, 0)],
         30: [("hold", 1, 1)], 31: [("hold", 0, 1)], 34: [("hold", 0, 0), ("hold", 1, 0)]}
# 8 -> 30 -> 8 fps (cap 16 -> 64 -> 16) while lane 0 is full, lane 1 warms (restarted at 18) and lane 2 is held (17..25)
FPS_EVENTS = {17: [("hold", 2, 1)], 18: [("restart", 1)], 26: [("hold", 2, 0)]}


def fps_steps(t):
    return 8.0 if t < 20 or t >= 30 else 30.0


SIZES = [(96, 64), (91, 67)]   # 91 x 67: the pyrUp chain ends at 92 x 68, so the bilinear resize runs


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("w,h", SIZES)
def test_restart_during_warmup_and_after_wrap(w, h, c):
    got = check_lanes(w, h, c, 3, 40, RESTARTS)
    assert list(got[5][2]) == [True, False, True]   # the restarted lane has one column: it does not produce


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("w,h", SIZES)
def test_holds_span_warmup_and_wrap(w, h, c):
    got = check_lanes(w, h, c, 3, 40, HOLDS)
    assert list(got[15][2]) == [True, True, False]


def test_three_lanes_restarted_at_different_frames():
    """lanes warm up at different lengths at once: one DFT pair per length per lane"""
    check_lanes(96, 64, 3, 4, 40, {7: [("restart", 0)], 12: [("restart", 2)], 20: [("restart", 3), ("hold", 1, 1)],
                                   23: [("hold", 1, 0)]})


@pytest.mark.parametrize("c", [3, 1])
def test_framerate_change_while_lanes_warm_run_and_hold(c):
    check_lanes(91, 67, c, 3, 44, FPS_EVENTS, fps=fps_steps)


@pytest.mark.skipif(EMU, reason="70 lanes of references are too slow for the CPU emulation")
def test_70_lanes_with_restarts():
    events = {6: [("restart", 0)], 10: [("restart", 64)], 19: [("restart", 69)]}
    got = run_lanes(64, 48, 3, 70, 24, events)
    want = references(64, 48, 3, 70, 24, events)
    for k in range(70):
        if k not in (0, 1, 63, 64, 65, 69):
            want[k] = []   # the lanes next to the restarted ones and the restarted ones themselves are checked
    assert_lanes_equal(got, want)


def test_option_off_keeps_the_refusal_and_lockstep_frames():
    """Without the option a hold is still refused; with it the same uniform frames give the same bytes."""
    cfg = color_cfg(8.0)
    a, b = proc(2), proc(2, LIFECYCLE)
    for t in range(20):
        f = stack(t, 2, 96, 64, 3)
        ra, rb = process_raw(a, f, cfg), process_raw(b, f, cfg)
        assert ra[0] == rb[0] and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2]), t
    a.hold_lane(1)
    with pytest.raises(L.MagcoreError) as e:
        process_raw(a, stack(20, 2, 96, 64, 3), cfg)
    assert e.value.status == capi.MC_ERR_UNSUPPORTED


def test_process_image_fills_idle_color_lanes_with_their_input():
    cfg = color_cfg(8.0)
    m = proc(3, LIFECYCLE)
    for t in range(4):
        if t == 3:
            m.restart_lane(0)
            m.hold_lane(2)
        f = stack(t, 3, 96, 64, 3)
        produced, out = m.process_image(f, cfg)
    assert produced and list(m.lane_produced()) == [False, True, False]
    assert np.array_equal(out[0], f[0]) and np.array_equal(out[2], f[2]) and not np.array_equal(out[1], f[1])


@pytest.mark.parametrize("pinned", [False, True])
def test_pipelined_submit_equals_blocking(pinned):
    """Restarts and holds are taken at submit time: three frames in flight give the blocking calls' frames and flags."""
    w, h, c, lanes, n, depth = 96, 64, 3, 4, 24, 3
    events = {3: [("hold", 3, 1)], 5: [("restart", 0)], 9: [("hold", 3, 0), ("restart", 2)],
              12: [("restart", 1), ("hold", 2, 1)], 19: [("hold", 2, 0)]}
    cfg = color_cfg(8.0)
    frames = [stack(t, lanes, w, h, c) for t in range(n)]
    a, b = proc(lanes, LIFECYCLE), proc(lanes, LIFECYCLE)
    ref = []
    for t in range(n):
        apply(a, events.get(t, []))
        ref.append(process_raw(a, frames[t], cfg))
    nbytes = frames[0].nbytes
    lib = capi.lib()
    if pinned:
        bufs = [lib.mc_host_alloc(nbytes) for _ in range(2 * n)]
        view = lambda p: np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=frames[0].shape)
        ins, outs = [view(p) for p in bufs[:n]], [view(p) for p in bufs[n:]]
        for t in range(n):
            ins[t][...] = frames[t]
    else:
        bufs, ins, outs = [], frames, [np.empty_like(frames[0]) for _ in range(n)]
    try:
        for o in outs:
            o[...] = SENTINEL
        got, done = [], 0
        for t in range(n):
            if t - done >= depth:
                got.append((b.collect(), b.lane_produced()))
                done += 1
            apply(b, events.get(t, []))
            b.submit(ins[t].ctypes.data, w, h, c, w * c, cfg, outs[t].ctypes.data, w * c)
        while done < n:
            got.append((b.collect(), b.lane_produced()))
            done += 1
        for t in range(n):
            assert got[t][0] == ref[t][0] and np.array_equal(got[t][1], ref[t][2]), t
            assert np.array_equal(outs[t], ref[t][1]), t
    finally:
        a.close()
        b.close()
        for p in bufs:
            lib.mc_host_free(p)


def test_clip_with_restart_and_hold_equals_frame_calls():
    """Restarts and holds are taken at the clip's first frame; a held lane is skipped for the whole clip."""
    from test_gpu_clip import clip_frames, run_clip, run_frames
    cfg = color_cfg(8.0)
    w, h, c, lanes = 96, 64, 3, 3
    a, b = proc(lanes, LIFECYCLE), proc(lanes, LIFECYCLE)
    t = 0
    for n, events in ((6, []), (5, [("restart", 1), ("hold", 2, 1)]), (7, [("hold", 2, 0)]), (20, [("restart", 0)])):
        fr = clip_frames(t, n, lanes, w, h, c)
        apply(a, events)
        apply(b, events)
        fa, oa = run_clip(a, fr, cfg)
        fb, ob = run_frames(b, fr, cfg)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob), (t, n)
        assert np.array_equal(a.lane_produced(), b.lane_produced())
        t += n
    a.close()
    b.close()


def test_chain_device_with_restarts_and_holds():
    from test_gpu_chain_lanes import check_chain
    steps = [("cfg", dict(down=2, roi=(0.1, 0.1, 0.8, 0.8), gray=True)), ("frame",), ("clip", 3), ("restart", 2),
             ("hold", 1, 1), ("frame",), ("clip", 4), ("hold", 1, 0), ("frame",), ("restart", 0), ("hold", 3, 1),
             ("clip", 2), ("hold", 3, 0), ("frame",)]
    check_chain(O.MODE_COLOR, COLOR_UI, 240, 180, 3, steps, lanes=4, options=LIFECYCLE, launches=True)


@pytest.mark.parametrize("settings", [dict(down=2, gray=True), dict(down=1)], ids=["front", "no_front"])
def test_nv12_chain_with_restarts_and_holds(settings):
    from test_gpu_chain_lanes import check_chain
    from test_gpu_nv12 import Layout
    steps = [("cfg", settings), ("frame",), ("clip", 3), ("hold", 1, 1), ("frame",), ("restart", 0), ("clip", 2),
             ("hold", 1, 0), ("frame",)]
    check_chain(O.MODE_COLOR, COLOR_UI, 130, 74, 3, steps, lanes=2, nv12=Layout(130, 74, pitch=133, uv_row=80),
                options=LIFECYCLE, launches=True)


@pytest.mark.parametrize("c", [3, 1])
def test_restarted_lane_against_the_oracle(c):
    """The restarted lane, from its restart on, is within Color's tolerances of a fresh oracle processor (pre-quantisation
    float output < 1e-4 of full scale, u8 <= 1 LSB)."""
    w, h, lanes, at, n, fps = 91, 67, 2, 9, 30, 8.0
    cfg, ocfg = make_cfgs(O.MODE_COLOR, *COLOR_UI, fps)
    m = proc(lanes, LIFECYCLE + (("keep_float_output", 1),))
    oproc = O.MagnificationProcessor()
    worst_f, worst_u8, checked = 0.0, 0, 0
    for t in range(n):
        if t == at:
            m.restart_lane(1)
        produced, out, flags = process_raw(m, stack(t, lanes, w, h, c), cfg)
        if t < at:
            continue
        dbg = {}
        oprod, oout = oproc.process(lane_frame(t, 1, w, h, c), ocfg, dbg)
        assert bool(flags[1]) == bool(oprod), t
        if not oprod:
            continue
        got = m.float_output(w, h, c)[1]
        ref = dbg["output_f32"] if c == 3 else dbg["output_f32"][..., None]
        worst_f = max(worst_f, float(np.abs(got - ref).max()) / 255.0)
        worst_u8 = max(worst_u8, int(u8_diff(out[1], oout).max()))
        checked += 1
    assert checked == n - at - 1
    assert worst_f < 1e-4 and worst_u8 <= 1, (worst_f, worst_u8)


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
def test_1080p_two_lane_restart_and_hold():
    events = {3: [("restart", 1)], 5: [("hold", 0, 1)], 7: [("hold", 0, 0)]}
    check_lanes(1920, 1080, 3, 2, 10, events, fps=lambda t: 30.0, ui=COLOR_UI[:5] + (3,))
