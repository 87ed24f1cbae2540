"""L-only synthesis of the Laplace path.  When the chroma factor is zero and the a / b motion is known to be finite, the
collapses and the strip egress synthesise the L planes only and take a and b from the input (DESIGN.md §4).  Every case
runs a default handle (strip egress: L-only wherever it applies) and a tile-egress handle (egress_strip = 0: always full
synthesis) on the same frames and requires bit-equal u8 frames and float taps."""
import ctypes as C
import math

import numpy as np
import pytest

from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_clip import clip_frames
from test_gpu_lanes import proc, process_raw, stack

pytestmark = pytest.mark.gpu


def params(chroma=0, levels=4, **raw):
    """mc_params from UI values; `raw` sets algorithm-unit fields afterwards (coLow, coHigh, amplification ...)"""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, chroma, levels)
    prm = _to_mc(cfg)
    for k, v in raw.items():
        setattr(prm, k, v)
    return prm


def pair(lanes=1, options=()):
    """(default handle, tile-egress handle), both keeping the float tap"""
    opts = tuple(options) + (("keep_float_output", 1),)
    return proc(lanes, opts), proc(lanes, opts + (("egress_strip", 0),))


def bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def step(a, b, frames, prm, tag):
    """one frame call on both handles: equal flags, u8 frames and float taps (bit for bit, NaN included)"""
    pa, oa, fa = process_raw(a, frames, prm)
    pb, ob, fb = process_raw(b, frames, prm)
    assert pa == pb and np.array_equal(fa, fb), tag
    assert np.array_equal(oa, ob), tag
    h, w = frames.shape[1:3]
    assert np.array_equal(bits(a.float_output(w, h, 3)), bits(b.float_output(w, h, 3))), tag


def check_shapes(w, h, lv, band_from_state, faithful=0, frames=4):
    a, b = pair(1, (("band_from_state", band_from_state), ("faithful_level0", faithful)))
    prm = params(levels=lv)
    for t in range(frames):
        step(a, b, stack(t, 1, w, h, 3), prm, (w, h, lv, band_from_state, t))


def check_lanes(w, h, lv, lanes=8, groups=2):
    """lane groups, then a restart and a hold, then the release"""
    a, b = pair(lanes, (("lane_groups", groups),))
    prm = params(levels=lv)
    for t in range(7):
        for p in (a, b):
            if t == 3:
                p.restart_lane(2)
                p.hold_lane(lanes - 3)
            if t == 5:
                p.hold_lane(lanes - 3, False)
        step(a, b, stack(t, lanes, w, h, 3), prm, t)


def run_clip_raw(p, frames, prm):
    n, lanes, h, w = frames.shape[:4]
    out = np.zeros_like(frames)
    flags = np.zeros((n, lanes), np.uint8)
    p._check(p._lib.mc_process_clip(p._h, frames.ctypes.data, n, w, h, 3, w * 3, C.byref(prm), out.ctypes.data, w * 3,
                                    flags.ctypes.data_as(C.POINTER(C.c_uint8))))
    return flags, out


def check_clips(w, h, lv, lanes=2, n=8, clips=2):
    """clips on the default handle equal frame calls on the default and on the tile-egress handle"""
    opts = (("keep_float_output", 1),)
    c, (a, b) = proc(lanes, opts), pair(lanes)
    prm = params(levels=lv)
    for k in range(clips):
        fr = clip_frames(k * n, n, lanes, w, h, 3)
        fc, oc = run_clip_raw(c, fr, prm)
        for t in range(n):
            pa, oa, fa = process_raw(a, fr[t], prm)
            pb, ob, fb = process_raw(b, fr[t], prm)
            assert np.array_equal(fc[t], fa.astype(np.uint8)) and np.array_equal(fa, fb), (k, t)
            assert np.array_equal(oc[t], oa) and np.array_equal(oa, ob), (k, t)
        tap = [bits(p.float_output(w, h, 3)) for p in (c, a, b)]
        assert np.array_equal(tap[0], tap[1]) and np.array_equal(tap[1], tap[2]), k
        for lvl in range(1, lv):
            for name in ("lowpassHi", "lowpassLo"):
                assert np.array_equal(c.get_state(name, lvl), b.get_state(name, lvl)), (k, lvl, name)


def check_chroma_switch(w, h, lv):
    """chroma 0 -> 30 -> 0: the a / b state keeps running while only L is synthesised"""
    a, b = pair()
    for t, chroma in enumerate((0, 0, 0, 30, 30, 0, 0, 30)):
        step(a, b, stack(t, 1, w, h, 3), params(chroma, lv), (t, chroma))


SENTINEL = np.float32(-12345.5)


def fill_band(p, lvl=1):
    r, c, ch = p.state_dims("band", lvl)
    p.set_state("band", lvl, np.full((p.lanes, ch, r, c), SENTINEL, np.float32))


def band_written(p, lvl=1):
    """after a frame whose band planes were filled with the sentinel: which planes it wrote ("L", "Lab" or "mixed")"""
    wr = (p.get_state("band", lvl) != SENTINEL).reshape(p.lanes, 3, -1)
    if wr[:, 0].all() and not wr[:, 1:].any():
        return "L"
    return "Lab" if wr.all() else "mixed"


def check_sticky_bound(w, h, lv):
    """Cutoffs outside [0, 1] turn L-only synthesis off until the state of every lane is dropped (mc_reset).  The band
    planes the level kernel stores (band_from_state 0) show which synthesis ran: under L-only synthesis their a / b
    planes are not written."""
    a, b = pair(1, (("band_from_state", 0),))
    good = params(levels=lv)
    t = 0

    def run(prm, probe=False):
        nonlocal t
        if probe:
            fill_band(a)
        step(a, b, stack(t, 1, w, h, 3), prm, t)
        t += 1
        return band_written(a) if probe else None

    run(good)
    assert run(good, probe=True) == "L"             # L-only
    for bad in (params(levels=lv, coHigh=1.5), params(levels=lv, coLow=-0.25)):
        run(bad)
    run(params(levels=lv, coHigh=math.nan))
    for _ in range(2):
        assert run(good, probe=True) == "Lab"          # full synthesis: the a / b state may be unbounded
    a.reset()
    b.reset()
    run(good)
    assert run(good, probe=True) == "L"             # L-only again
    # a per-lane restart does not drop every lane's state
    m, n = pair(2, (("band_from_state", 0),))
    for k, prm in enumerate((good, good, params(levels=lv, coHigh=2.0), good)):
        step(m, n, stack(t + k, 2, w, h, 3), prm, ("lanes", k))
    for p in (m, n):
        p.restart_lane(0)
        p.restart_lane(1)
    step(m, n, stack(t + 4, 2, w, h, 3), good, "restarted")
    fill_band(m)
    step(m, n, stack(t + 5, 2, w, h, 3), good, "after restart")
    assert band_written(m) == "Lab"


def check_huge_gains(w, h, lv):
    """amplification 1e38 and inf at chroma 0 (gains beyond 2^64 or not finite: full synthesis)"""
    for amp in (1e38, math.inf):
        a, b = pair()
        for t in range(4):
            step(a, b, stack(t, 1, w, h, 3), params(levels=lv, amplification=amp), (amp, t))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("band_from_state", [1, 0])
@pytest.mark.parametrize("w,h,lv", [(640, 480, 4), (333, 251, 5), (121, 75, 3), (119, 64, 3), (240, 67, 2), (250, 131, 2),
                                    (481, 270, 6), (126, 129, 3)])
def test_luma_synthesis_equals_full_synthesis(w, h, lv, band_from_state):
    check_shapes(w, h, lv, band_from_state)


@pytest.mark.parametrize("band_from_state", [1, 0])
def test_luma_synthesis_faithful_level0(band_from_state):
    check_shapes(333, 251, 5, band_from_state, faithful=1)


def test_luma_synthesis_1080p():
    check_shapes(1920, 1080, 6, 1, frames=3)


def test_luma_synthesis_lanes_restart_hold():
    check_lanes(200, 136, 4)


def test_luma_synthesis_clips():
    check_clips(333, 251, 5)


def test_luma_synthesis_chroma_switch():
    check_chroma_switch(333, 251, 5)


def test_luma_synthesis_sticky_bound():
    check_sticky_bound(200, 136, 4)


def test_luma_synthesis_huge_gains():
    check_huge_gains(200, 136, 4)
