"""Labels on the device export canvas (mc_set_overlay): every compose call maps its canvases through the handle's overlay.

The checkers of test_gpu_compose.py and test_gpu_yuv422.py run unchanged under `overlaid(make)`: every handle they
create gets the overlay make(cw, ch) for each canvas geometry before the call that uses it, and their expected canvas
becomes Overlay.apply(compose(...)) (and its NV12 conversion for NV12 canvases).  So the flags, info, lane flags, state
afterwards and the single "compose" launch are still checked against the twin handle, whose chain calls must ignore
the overlay it also carries.  Overlays are the exporter's real labels (lvm_b200.labels) or synthetic rects with random
maps at odd columns and rows, 1 x 1, the whole canvas, across the left/right seam and on the last row and column."""
import ctypes as C
import os
from contextlib import contextmanager

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.labels import Overlay, export_labels
from oracle import livim_oracle as O
import test_gpu_compose as TC
import test_gpu_yuv422 as TY
from compose_oracle import compose
from test_gpu_chain_lanes import MODES, chain_cfg
from test_gpu_compose import SPLITS, Canvas, check_compose, sources
from test_gpu_lanes import LAPLACE_UI, SENTINEL, state_names
from test_gpu_nv12 import Dev

EMU = os.environ.get("MC_EMU") == "1"
pytestmark = pytest.mark.gpu

W, H = (66, 38) if EMU else (134, 78)
LR, TB = capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM


@contextmanager
def overlaid(make):
    """Within: every ProcessingChainB200 created gets make(cw, ch) whenever compose_geometry reports a new non-empty
    canvas, and the checkers' compose() applies it."""
    handles, cur = [], {}
    chain, geom = L.ProcessingChainB200, L.MagnificationProcessor.compose_geometry
    saved = (TC.compose, TY.compose)

    def new_chain(*args, **kw):
        ch = chain(*args, **kw)
        handles.append(ch)
        return ch

    def new_geom(cfg, w, h, c, split):
        cw, chh = geom(cfg, w, h, c, split)
        if cw and cur.get("geom") != (cw, chh):
            cur["geom"], cur["ov"] = (cw, chh), make(cw, chh)
            for ch in handles:
                ch.magnifier.set_overlay(cur["ov"])
        return cw, chh

    def labelled(original, proc, split):
        im = compose(original, proc, split)
        return None if im is None else cur["ov"].apply(im)

    L.ProcessingChainB200 = new_chain
    L.MagnificationProcessor.compose_geometry = staticmethod(new_geom)
    TC.compose = TY.compose = labelled
    try:
        yield cur
    finally:
        L.ProcessingChainB200 = chain
        L.MagnificationProcessor.compose_geometry = staticmethod(geom)
        TC.compose, TY.compose = saved


def labels(cw, ch, split):
    return export_labels(cw, ch, split)


def synthetic(kind, seed=0):
    """-> make(cw, ch): random maps on rects of the given kind"""
    def make(cw, ch):
        rng = np.random.default_rng(seed + cw * 7 + ch)
        if kind == "odd":              # odd starts and ends; the second ends on the last row and column
            boxes = [(3, 1, min(13, cw - 3), min(5, ch - 1)), (cw - 7, ch - 3, 7, 3)]
        elif kind == "pixel_seam":     # one pixel, and a band across the middle column (the left/right seam)
            boxes = [(1, ch - 1, 1, 1), (cw // 2 - 5, 1, 11, ch - 2)]
        else:                          # the whole canvas
            boxes = [(0, 0, cw, ch)]
        maps = 300
        rects = [(x, y, rng.integers(0, maps, (h, w), dtype=np.uint16)) for x, y, w, h in boxes]
        return Overlay(cw, ch, rects, rng.integers(0, 256, (maps, 256), dtype=np.uint8))
    return make


# ---- sources, canvases, lanes and clips ----------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", [capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12], ids=["bgr_canvas", "nv12_canvas"])
@pytest.mark.parametrize("src", ["bgr", "gray", "nv12"])
@pytest.mark.parametrize("gray", [False, True], ids=["color", "grayscale"])
@pytest.mark.parametrize("split", list(SPLITS))
def test_labels_on_every_source_and_canvas(split, gray, src, fmt):
    """Real labels through no front stage, a ROI and a downscale (each a new geometry and overlay); frames and clips"""
    steps = [("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 3), ("cfg", dict(down=2)), ("frame",),
             ("clip", 2)]
    with overlaid(lambda cw, ch: labels(cw, ch, SPLITS[split])):
        check_compose(O.MODE_LAPLACE, LAPLACE_UI, W, H, src, fmt, SPLITS[split], steps, lanes=2, gray=gray, pad=5,
                      lane_rows=1, uv_gap=3)


@pytest.mark.parametrize("fmt", [capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12], ids=["bgr_canvas", "nv12_canvas"])
@pytest.mark.parametrize("gray", [False, True], ids=["color", "grayscale"])
@pytest.mark.parametrize("split", [LR, TB], ids=["left_right", "top_bottom"])
def test_labels_on_yuyv_sources(split, gray, fmt):
    steps = [("frame",), ("cfg", dict(down=2)), ("clip", 3)]
    with overlaid(lambda cw, ch: labels(cw, ch, split)):
        TY.check_compose_yuv(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, split, steps, lanes=2, gray=gray, pad=5,
                             lane_rows=1, uv_gap=3)


@pytest.mark.parametrize("kind", ["odd", "pixel_seam", "whole"])
@pytest.mark.parametrize("src", ["bgr", "nv12"])
@pytest.mark.parametrize("fmt", [capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12], ids=["bgr_canvas", "nv12_canvas"])
def test_synthetic_overlays(kind, src, fmt):
    """Random maps on rects with odd edges (cutting NV12 2x2 blocks), 1 x 1, across the seam, on the last row and column,
    and over the whole canvas; padded pitches and lane strides"""
    for split in (LR, TB, capi.MC_SPLIT_NONE):
        with overlaid(synthetic(kind)):
            check_compose(O.MODE_LAPLACE, LAPLACE_UI, W, H, src, fmt, split, [("frame",), ("cfg", dict(down=2)), ("clip", 2)],
                          lanes=2, pad=5, lane_rows=1, uv_gap=3, in_pad=2)


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_lanes_with_hold_and_restart(mname):
    """3 lanes, one held and one restarted mid-clip: held lanes' canvases stay sentinel"""
    mode, ui = MODES[mname]
    steps = [("cfg", dict(down=2, roi=(0.05, 0.0, 0.9, 1.0))), ("clip", 2), ("hold", 1, 1), ("restart", 2), ("clip", 3),
             ("frame",), ("hold", 1, 0), ("restart", 0), ("clip", 2)]
    with overlaid(synthetic("odd", 3)):
        check_compose(mode, ui, W, H, "nv12", capi.MC_CANVAS_NV12, LR, steps, lanes=3, pad=3, lane_rows=2, uv_gap=1, in_pad=2)


@pytest.mark.parametrize("fmt", [capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12], ids=["bgr_canvas", "nv12_canvas"])
def test_aligned_canvases_and_mode_none(fmt):
    """8-byte aligned rows take the 64-bit path around the mapped pixels; mode None writes a canvas every frame"""
    for split in (LR, TB):
        with overlaid(synthetic("pixel_seam", 5)):
            check_compose(O.MODE_NONE, LAPLACE_UI, 64, 32, "bgr", fmt, split, [("frame",), ("clip", 2)], lanes=2)
        with overlaid(lambda cw, ch: labels(cw, ch, split)):
            check_compose(O.MODE_LAPLACE, LAPLACE_UI, 64, 32, "nv12", fmt, split, [("frame",), ("clip", 2)], lanes=2, pad=8)


@pytest.mark.skipif(EMU, reason="wide frames are too slow for the CPU emulation")
@pytest.mark.parametrize("w,h,split", [(640, 96, LR), (1280, 64, TB), (1200, 40, LR)],
                         ids=["thickness1", "thickness2_tb", "thickness2_lr"])
def test_real_labels_at_wider_panes(w, h, split):
    with overlaid(lambda cw, ch: labels(cw, ch, split)):
        check_compose(O.MODE_LAPLACE, LAPLACE_UI, w, h, "bgr", capi.MC_CANVAS_NV12, split, [("frame",), ("clip", 2)],
                      lanes=2, pad=8)


@pytest.mark.skipif(EMU, reason="1080p frames are too slow for the CPU emulation")
def test_1080p_left_right_into_nv12():
    with overlaid(lambda cw, ch: labels(cw, ch, LR)):
        check_compose(O.MODE_LAPLACE, LAPLACE_UI, 1920, 1080, "nv12", capi.MC_CANVAS_NV12, LR, [("frame",), ("clip", 2)],
                      lanes=2, pad=64, uv_gap=8)


# ---- clearing, resets and errors ------------------------------------------------------------------------------------

def _canvas_after(m, cfg, data, split, fmt=capi.MC_CANVAS_NV12, lanes=2):
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, split)
    cv = Canvas(fmt, cw, ch, lanes, pad=3)
    st = _raw(m, cfg, data, split, cv.struct())
    m.sync()
    return st, cv.dev.numpy()


def _raw(m, cfg, data, split, canvas):
    from lvm_b200.processor import _to_mc
    p, info = _to_mc(cfg), capi.McChainInfo()
    d_in = Dev(np.ascontiguousarray(data))
    flags = np.zeros(len(data), np.uint8)
    m._keep = d_in   # the input stays allocated until the caller's sync
    return capi.lib().mc_chain_compose_device(m._h, d_in.ptr, 1, W, H, 3, 3 * W, C.byref(p), 0, split, C.byref(canvas),
                                              flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(info))


def test_clear_and_reset():
    """After clear_overlay the canvases are those of a handle that never had one; the overlay survives mc_reset"""
    cfg = chain_cfg(O.MODE_LAPLACE, LAPLACE_UI)
    a, b = L.ProcessingChainB200(0, lanes=2).magnifier, L.ProcessingChainB200(0, lanes=2).magnifier
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, LR)
    ov = synthetic("whole", 9)(cw, ch)
    a.set_overlay(ov)
    for t in range(2):
        data, _ = sources(t, 1, 2, W, H, "bgr")
        sa, ca = _canvas_after(a, cfg, data, LR)
        sb, cb = _canvas_after(b, cfg, data, LR)
        assert sa == sb == capi.MC_OK and not np.array_equal(ca, cb)
    a.reset()
    b.reset()
    data, _ = sources(2, 1, 2, W, H, "bgr")
    _, ca = _canvas_after(a, cfg, data, LR, fmt=capi.MC_CANVAS_BGR)
    _, cb = _canvas_after(b, cfg, data, LR, fmt=capi.MC_CANVAS_BGR)
    plain = cb[:, :ch, :3 * cw].reshape(2, ch, cw, 3)
    assert np.array_equal(ca[:, :ch, :3 * cw].reshape(2, ch, cw, 3), np.stack([ov.apply(x) for x in plain]))
    a.clear_overlay()
    data, _ = sources(3, 1, 2, W, H, "bgr")
    assert np.array_equal(_canvas_after(a, cfg, data, LR)[1], _canvas_after(b, cfg, data, LR)[1])


def test_errors_keep_the_previous_overlay_and_return_before_any_launch():
    cfg = chain_cfg(O.MODE_LAPLACE, LAPLACE_UI)
    m = L.ProcessingChainB200(0, lanes=2).magnifier
    lib = capi.lib()
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, LR)
    good = synthetic("odd", 11)(cw, ch)
    m.set_overlay(good)
    idx = np.zeros((4, 4), np.uint16)
    pal = np.zeros((2, 256), np.uint8)

    def ov(cw_=cw, ch_=ch, rects=((1, 1, idx),), palette=pal, **field):
        o = Overlay(cw_, ch_, list(rects), palette)
        for k, v in field.items():
            setattr(o.struct, k, v)
        return o

    bad = [ov(cw_=0), ov(ch_=0), ov(rects=((cw - 3, 0, idx),)), ov(rects=((0, ch - 2, idx),)), ov(rects=((-1, 0, idx),)),
           ov(rects=((0, 0, idx), (3, 3, idx))), ov(rects=((0, 0, np.full((4, 4), 2, np.uint16)),)), ov(maps=0),
           ov(maps=65537), ov(map=None)]
    for field, value in (("rects", 3), ("rects", -1)):
        o = ov()
        setattr(o.struct, field, value)
        bad.append(o)
    o = ov()
    o.struct.rect[0].index = None
    bad.append(o)
    o = ov()
    o.struct.rect[0].w = 0
    bad.append(o)
    for b in bad:
        assert lib.mc_set_overlay(m._h, C.byref(b.struct)) == capi.MC_ERR_INVALID, b.struct
    data, _ = sources(0, 1, 2, W, H, "bgr")
    twin = L.ProcessingChainB200(0, lanes=2).magnifier
    st, got = _canvas_after(m, cfg, data, LR, fmt=capi.MC_CANVAS_BGR)
    _, plain = _canvas_after(twin, cfg, data, LR, fmt=capi.MC_CANVAS_BGR)
    assert st == capi.MC_OK
    assert np.array_equal(got[:, :ch, :3 * cw].reshape(2, ch, cw, 3),
                          np.stack([good.apply(x) for x in plain[:, :ch, :3 * cw].reshape(2, ch, cw, 3)]))
    # a canvas of another geometry: refused before any launch, canvases and state untouched
    m.set_overlay(synthetic("odd")(cw + 2, ch))
    before, n0 = [m.get_state(n, l) for n, l in state_names(m, O.MODE_LAPLACE)], m.launch_count
    for split in (LR, TB):
        st, buf = _canvas_after(m, cfg, data, split)
        assert st == capi.MC_ERR_INVALID and (buf == SENTINEL).all()
    assert m.launch_count == n0
    assert all(np.array_equal(m.get_state(n, l), a) for (n, l), a in zip(state_names(m, O.MODE_LAPLACE), before))
    # an empty (0 x 0) canvas with an overlay set is no mismatch: the chain runs, nothing is composed
    empty = chain_cfg(O.MODE_LAPLACE, LAPLACE_UI, roi=(0.0, 0.0, 1.0, 0.01))
    assert _canvas_after(m, empty, data, LR)[0] == capi.MC_OK
