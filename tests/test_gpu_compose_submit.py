"""The export canvas from host clips, pipelined (mc_chain_compose_submit, _nv12 and _yuv422, collected by mc_collect).

Every case runs a twin handle that calls the matching device compose call (mc_chain_compose_device or its _nv12 /
_yuv422 form) on device copies of the same host clips, into sentinel-filled canvases of the same layout, and must equal
it bit for bit: every canvas byte (row padding, spare lane rows, a detached NV12 chroma plane and held lanes included),
the [frames][lanes] flags of every collect, *produced and mc_lane_produced after each collect, the info of every submit
(magnified 0) and the state planes at the end.  Restarts, holds, a lane-params change, a ROI move, a levels change and
an overlay set / replace / clear happen while clips are in flight; clips of 16, 3 and 1 frames share the slots, and the
last, shorter clip goes in while longer ones are in flight.  Compose submits interleave with mc_submit and
mc_chain_submit_yuv422 in FIFO order, and every bad submit returns before any launch with the clips in flight unchanged."""
import ctypes as C
import dataclasses
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.labels import export_labels
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_chain_lanes import MODES, chain_cfg
from test_gpu_chain_submit import ORDER, Source, host_buffer, info_tuple
from test_gpu_compose import Canvas
from test_gpu_compose_labels import synthetic
from test_gpu_lanes import SENTINEL, lane_frame, state_names
from test_gpu_nv12 import Dev, Layout, to_nv12
from test_gpu_yuv422 import Yuv, from_bgr

pytestmark = pytest.mark.gpu

EMU = os.environ.get("MC_EMU") == "1"
W, H = (66, 38) if EMU else (134, 78)
ROI, ROI_MOVED = (0.1, 0.15, 0.7, 0.75), (0.2, 0.05, 0.7, 0.75)
FRONTS = {"none": {}, "roi": dict(roi=ROI), "down2": dict(down=2), "gray": dict(gray=True)}
SOURCES = ("bgr", "gray", "nv12", "yuyv", "uyvy")
BGR, NV12 = capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12
NONE, LR, TB = capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM
CLIPS = (16, 3, 1, 16, 3, 1, 16, 5)   # the first sizes the slots; the last, shorter one goes in while others are in flight


class ClipSource:
    """Clips of one source kind: frames t0 .. t0 + n - 1 of every lane as one host buffer, virtual lane (t - t0) * lanes
    + k, with padded rows (NV12: a Cb,Cr plane that does not follow the luma plane; 4:2:2: spare rows after each frame)."""

    def __init__(self, kind, lanes, w, h, pad):
        self.kind, self.lanes, self.w, self.h = kind, lanes, w, h
        self.c = 1 if kind == "gray" else 3
        self.in_step = w * self.c + pad
        if kind == "nv12":
            self.lay = Layout(w, h, pitch=w + pad, uv_row=h + (4 if pad else 0))
        elif kind in ORDER:
            self.lay = Yuv(w, h, ORDER[kind], pitch=2 * w + pad, lane_rows=2 if pad else 0)

    def pack(self, bgr):
        """[V] BGR frames -> the host buffer of this kind"""
        if self.kind == "nv12":
            return self.lay.pack(np.stack([to_nv12(f) for f in bgr]), fill=0x3C)
        if self.kind in ORDER:
            return self.lay.pack(np.stack([from_bgr(f, ORDER[self.kind]) for f in bgr]))
        img = np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]) if self.c == 1 else np.stack(bgr)
        buf = np.full((len(bgr), self.h, self.in_step), 0x3C, np.uint8)
        buf[:, :, :self.w * self.c] = img.reshape(len(bgr), self.h, self.w * self.c)
        return buf

    def clip(self, t0, n):
        return self.pack([lane_frame(t, k, self.w, self.h, 3) for t in range(t0, t0 + n) for k in range(self.lanes)])

    def device_call(self, m, cfg, d_in, n, split, canvas):
        w, h = self.w, self.h
        if self.kind == "nv12":
            return m.chain_compose_nv12_device(self.lay.planes(d_in), n, w, h, cfg, split, canvas)
        if self.kind in ORDER:
            return m.chain_compose_yuv422_device(self.lay.struct(d_in), n, w, h, cfg, split, canvas)
        return m.chain_compose_device(d_in, n, w, h, self.c, self.in_step, cfg, split, canvas)

    def submit(self, ch, cfg, base, n, split, canvas):
        w, h = self.w, self.h
        if self.kind == "nv12":
            return ch.compose_submit_nv12(self.lay.planes(base), n, w, h, cfg, split, canvas)
        if self.kind in ORDER:
            return ch.compose_submit_yuv422(self.lay.struct(base), n, w, h, cfg, split, canvas)
        return ch.compose_submit(base, n, w, h, self.c, self.in_step, cfg, split, canvas)


def host_canvas(cv, pinned, lib, keep):
    """a sentinel-filled host copy of Canvas cv's layout, and its McCanvas"""
    buf = host_buffer(cv.dev.numpy().shape, pinned, lib, keep, SENTINEL)
    base = buf.ctypes.data
    return buf, cv.struct(data=base, uv=base + cv.uv_row * cv.pitch if cv.uv_row is not None else None)


def events_for(lanes, n):
    """{submit: [event]} between submits, with clips in flight: an overlay set, a restart and a lane-params change, a hold
    and its release, an overlay clear with a ROI move, the labels of the new geometry, a replaced overlay, a levels
    change.  Chain settings come before overlays, which are built for the geometry after them."""
    last, held = lanes - 1, min(1, lanes - 1)
    ev = {1: [("overlay", "labels")], 2: [("restart", last), ("lane_params", 0)], 3: [("hold", held, 1)],
          4: [("hold", held, 0), ("roi", ROI_MOVED), ("overlay", None)], 5: [("overlay", "labels")],
          6: [("overlay", "synthetic"), ("levels", 2)]}
    return {t: e for t, e in ev.items() if t < n}


def apply(chains, cfg, evs, held, geom):
    for e in evs:
        if e[0] == "restart":
            for ch in chains:
                ch.magnifier.restart_lane(e[1])
        elif e[0] == "hold":
            for ch in chains:
                ch.magnifier.hold_lane(e[1], bool(e[2]))
            held[e[1]] = bool(e[2])
        elif e[0] == "lane_params":
            lp = dataclasses.replace(cfg.magnification, amplification=cfg.magnification.amplification * 0.5 + 3)
            for ch in chains:
                ch.set_lane_params(e[1], lp)
        elif e[0] == "roi":
            cfg.preprocess.roiEnabled = True
            cfg.preprocess.roiX, cfg.preprocess.roiY, cfg.preprocess.roiW, cfg.preprocess.roiH = e[1]
        elif e[0] == "levels":
            cfg.magnification.levels = e[1]
        elif e[0] == "overlay":
            cw, chh, split = geom()
            ov = None if e[1] is None or not cw else export_labels(cw, chh, split) if e[1] == "labels" else synthetic("whole")(cw, chh)
            for ch in chains:
                ch.magnifier.set_overlay(ov) if ov is not None else ch.magnifier.clear_overlay()


def check_compose_submit(kind, front, mname, lanes=1, depth=3, clips=CLIPS, fmt=BGR, split=LR,
                         pins=((True, False), (False, True)), pad=6, lane_rows=1, uv_gap=3, events=None, w=W, h=H):
    """Clips of `kind` through the compose submits of one handle (pipeline_depth `depth`; pins: (input, canvas) pinned,
    cycled over the submits) against the twin's device compose calls."""
    mode, ui = MODES[mname]
    cfg = chain_cfg(mode, ui, **FRONTS[front])
    src = ClipSource(kind, lanes, w, h, pad)
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    if mode == O.MODE_COLOR and lanes > 1:
        for ch in (sub, twin):
            ch.magnifier.set_option("color_lane_lifecycle", 1)
    sub.magnifier.set_option("pipeline_depth", depth)
    evs = events_for(lanes, len(clips)) if events is None else events
    lib, keep = capi.lib(), []
    held = [False] * lanes
    pending, last = [], [np.zeros(lanes, bool)]

    def geom():
        return (*L.MagnificationProcessor.compose_geometry(cfg, w, h, src.c, split), split)

    def collect_one():
        ref, canvas, _, flags = pending.pop(0)
        assert np.array_equal(sub.magnifier.lane_produced(), last[0])   # unchanged until the clip is collected
        assert sub.magnifier.collect() == bool(ref["flags"].any()), ref["i"]
        assert np.array_equal(flags, ref["flags"]), (ref["i"], flags, ref["flags"])
        assert np.array_equal(sub.magnifier.lane_produced(), ref["lane_produced"]), ref["i"]
        assert np.array_equal(canvas, ref["canvas"]), (ref["i"], np.argwhere(canvas != ref["canvas"])[:5])
        for v in range(canvas.shape[0]):
            if ref["held"][v % lanes] or ref["empty"]:
                assert (canvas[v] == SENTINEL).all(), (ref["i"], v)
        last[0] = ref["lane_produced"]

    try:
        t = 0
        for i, n in enumerate(clips):
            apply((sub, twin), cfg, evs.get(i, []), held, geom)
            frames = src.clip(t, n)
            t += n
            cw, chh, _ = geom()
            cv = Canvas(fmt, cw, chh, n * lanes, pad, lane_rows, uv_gap)
            d_in = Dev(frames)
            tflags, tinfo = src.device_call(twin.magnifier, cfg, d_in.ptr, n, split, cv.struct())
            twin.magnifier.sync()
            ref = dict(i=i, flags=tflags.astype(np.uint8), lane_produced=twin.magnifier.lane_produced(), canvas=cv.dev.numpy(),
                       held=list(held), empty=cw == 0)
            if len(pending) == depth:
                collect_one()
            pin_in, pin_cv = pins[i % len(pins)]
            host_in = host_buffer(frames.shape, pin_in, lib, keep, 0)
            host_in[...] = frames
            canvas, mc = host_canvas(cv, pin_cv, lib, keep)
            info, flags = src.submit(sub, cfg, host_in.ctypes.data, n, split, mc)
            assert flags.shape == (n, lanes)
            assert info_tuple(info) == info_tuple(tinfo)[:-1] + (0,), i
            pending.append((ref, canvas, host_in, flags))   # every buffer stays valid until its clip is collected
        while pending:
            collect_one()
        for name, level in state_names(twin.magnifier, mode):
            assert np.array_equal(sub.magnifier.get_state(name, level), twin.magnifier.get_state(name, level)), (name, level)
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)


# ---- sources x fronts, canvases and splits ----------------------------------------------------------------------------

@pytest.mark.parametrize("front", list(FRONTS))
@pytest.mark.parametrize("kind", SOURCES)
def test_sources_and_fronts_equal_the_device_compose(kind, front):
    i = SOURCES.index(kind) + list(FRONTS).index(front)
    fmt, split = [(BGR, LR), (NV12, TB), (NV12, LR), (BGR, NONE), (NV12, NONE), (BGR, TB)][i % 6]
    check_compose_submit(kind, front, "laplace", lanes=3, depth=3, fmt=fmt, split=split)


@pytest.mark.parametrize("fmt", [BGR, NV12], ids=["bgr_canvas", "nv12_canvas"])
@pytest.mark.parametrize("split", [NONE, LR, TB], ids=["none", "left_right", "top_bottom"])
def test_splits_and_canvas_formats(split, fmt):
    check_compose_submit("nv12", "down2", "laplace", lanes=1, depth=3, fmt=fmt, split=split, pad=3, lane_rows=2, uv_gap=1)


# ---- modes x lanes x pipeline depths -----------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [1, 3, 5])
@pytest.mark.parametrize("lanes", [1, 3])
@pytest.mark.parametrize("mname", ["laplace", "phase", "color"])
def test_modes_lanes_and_depths(mname, lanes, depth):
    kind = ["bgr", "yuyv", "nv12"][depth // 2]
    front = ["roi", "down2", "gray"][depth // 2]
    fmt = NV12 if lanes == 1 else BGR
    check_compose_submit(kind, front, mname, lanes=lanes, depth=depth, fmt=fmt, split=LR)


@pytest.mark.parametrize("pins", [((False, False),), ((True, False),), ((False, True),), ((True, True),)],
                         ids=["pageable", "pinned_in", "pinned_canvas", "pinned_both"])
@pytest.mark.parametrize("pad", [0, 6], ids=["tight", "padded"])
def test_pinned_and_pageable_buffers(pins, pad):
    check_compose_submit("yuyv", "roi", "phase", lanes=3, depth=3, fmt=NV12, split=TB, pins=pins, pad=pad,
                         lane_rows=pad // 3, uv_gap=pad // 2)


# ---- FIFO with the other submits ---------------------------------------------------------------------------------------

def check_interleaved(w, h, lanes=2, n=12, pinned=False):
    """mc_submit, mc_chain_submit_yuv422 and compose submits of clips in turn on one handle: each collect equals its own
    call on a twin handle that runs the device calls in the same order"""
    mode, ui = MODES["laplace"]
    cfg = chain_cfg(mode, ui)   # one geometry: the calls share the temporal state without a structural reset
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    yv = Source("yuyv", lanes, w, h, 4)
    cs = ClipSource("bgr", lanes, w, h, 2)
    lib, keep, pending, ref = capi.lib(), [], [], []
    t = 0
    try:
        for i in range(n):
            which = ("compose", "submit", "chain_yuyv")[i % 3]
            if which == "submit":
                x = np.stack([lane_frame(t, k, w, h, 3) for k in range(lanes)])
                t += 1
                d_in, d_out = Dev(x), Dev(np.full_like(x, SENTINEL))
                twin.magnifier.process_device(d_in.ptr, w, h, 3, 3 * w, cfg, d_out.ptr, 3 * w)
                host_in, out = host_buffer(x.shape, pinned, lib, keep, 0), host_buffer(x.shape, pinned, lib, keep, SENTINEL)
                host_in[...] = x
                sub.magnifier.submit(host_in.ctypes.data, w, h, 3, 3 * w, cfg, out.ctypes.data, 3 * w)
                outs, want, flags = (out,), (d_out,), None
            elif which == "chain_yuyv":
                frame = yv.frame(t)
                t += 1
                (oh, orow), (gh, grow), _ = yv.geometry(cfg)
                d_in = Dev(frame)
                d_out, d_orig = Dev(np.full((lanes, oh, orow), SENTINEL, np.uint8)), Dev(np.full((lanes, gh, grow), SENTINEL, np.uint8))
                yv.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
                host_in = host_buffer(frame.shape, pinned, lib, keep, 0)
                host_in[...] = frame
                out = host_buffer((lanes, oh, orow), pinned, lib, keep, SENTINEL)
                orig = host_buffer((lanes, gh, grow), pinned, lib, keep, SENTINEL)
                yv.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, orow, orig.ctypes.data, grow)
                outs, want, flags = (out, orig), (d_out, d_orig), None
            else:
                nf = 3
                frames = cs.clip(t, nf)
                t += nf
                cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
                cv = Canvas(NV12, cw, chh, nf * lanes, 2, 1, 2)
                d_in = Dev(frames)
                cs.device_call(twin.magnifier, cfg, d_in.ptr, nf, LR, cv.struct())
                host_in = host_buffer(frames.shape, pinned, lib, keep, 0)
                host_in[...] = frames
                canvas, mc = host_canvas(cv, pinned, lib, keep)
                _, flags = cs.submit(sub, cfg, host_in.ctypes.data, nf, LR, mc)
                outs, want = (canvas,), (cv.dev,)
            twin.magnifier.sync()
            ref.append((which, twin.magnifier.lane_produced(), tuple(d.numpy() for d in want)))
            pending.append((outs, host_in, flags))
            if len(pending) == 3 or i < 3:   # the slots grow to the clip while nothing is in flight
                _collect_and_compare(sub, ref, pending)
        while pending:
            _collect_and_compare(sub, ref, pending)
        for name, level in state_names(twin.magnifier, mode):
            assert np.array_equal(sub.magnifier.get_state(name, level), twin.magnifier.get_state(name, level)), (name, level)
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)


def _collect_and_compare(sub, ref, pending):
    i = len(ref) - len(pending)
    which, lane_prod, want = ref[i]
    outs, _, flags = pending.pop(0)
    sub.magnifier.collect()
    assert np.array_equal(sub.magnifier.lane_produced(), lane_prod), (i, which)
    if flags is not None:
        assert np.array_equal(flags[-1].astype(bool), lane_prod), (i, which)
    for got, exp in zip(outs, want):
        assert np.array_equal(got, exp), (i, which)


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_every_submit_interleaves_in_fifo_order(pinned):
    check_interleaved(W, H, pinned=pinned)


# ---- errors ------------------------------------------------------------------------------------------------------------

def check_errors(w, h, lanes=2):
    """Every bad compose submit returns its code with the launch count unchanged and no canvas written; the clips in
    flight are then collected equal to the twin's device calls.  The device clip calls refuse while they are in flight."""
    mode, ui = MODES["laplace"]
    cfg = chain_cfg(mode, ui, down=2, roi=ROI)
    lib, p = capi.lib(), _to_mc(cfg)
    ch, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    m = ch.magnifier
    m.set_option("pipeline_depth", 2)
    src, nvs, yvs = ClipSource("bgr", lanes, w, h, 0), ClipSource("nv12", lanes, w, h, 4), ClipSource("yuyv", lanes, w, h, 4)
    n = 3
    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
    clips = [src.clip(n * t, n) for t in range(3)]
    cvs = [Canvas(BGR, cw, chh, n * lanes, 2) for _ in range(3)]
    want = []
    for t in range(2):
        d_in = Dev(clips[t])
        flags, _ = src.device_call(twin.magnifier, cfg, d_in.ptr, n, LR, cvs[t].struct())
        twin.magnifier.sync()
        want.append((flags.astype(np.uint8), cvs[t].dev.numpy(), twin.magnifier.lane_produced()))
    keep = []
    canvases = [host_canvas(cv, False, lib, keep) for cv in cvs]
    _, flags0 = src.submit(ch, cfg, clips[0].ctypes.data, n, LR, canvases[0][1])
    spare, spare_cv = host_canvas(cvs[2], False, lib, keep)
    prod = np.zeros(64 * lanes, np.uint8)
    ok = dict(in_=clips[1].ctypes.data, frames=n, w=w, h=h, c=3, in_step=3 * w, p=p, gray=0, split=LR, canvas=spare_cv,
              produced=prod.ctypes.data_as(C.POINTER(C.c_uint8)), info=capi.McChainInfo())

    def bgr(**kw):
        a = {**ok, **kw}
        return lib.mc_chain_compose_submit(m._h, a["in_"], a["frames"], a["w"], a["h"], a["c"], a["in_step"], a["p"] and C.byref(a["p"]),
                                           a["gray"], a["split"], a["canvas"] and C.byref(a["canvas"]), a["produced"],
                                           a["info"] and C.byref(a["info"]))

    nvf, yvf = nvs.clip(0, n), yvs.clip(0, n)
    nvp, yst = nvs.lay.planes(nvf.ctypes.data), yvs.lay.struct(yvf.ctypes.data)

    def nv12(planes, ww=w, canvas=spare_cv):
        return lib.mc_chain_compose_submit_nv12(m._h, planes and C.byref(planes), n, ww, h, C.byref(p), 0, LR, C.byref(canvas),
                                                ok["produced"], C.byref(capi.McChainInfo()))

    def yuv(frame, ww=w):
        return lib.mc_chain_compose_submit_yuv422(m._h, frame and C.byref(frame), n, ww, h, C.byref(p), 0, LR, C.byref(spare_cv),
                                                  ok["produced"], C.byref(capi.McChainInfo()))

    bad_mode = _to_mc(cfg)
    bad_mode.mode = 7
    c0 = spare_cv
    nv_canvas = capi.McCanvas(NV12, c0.data, None, c0.pitch, c0.lane_stride)
    n0 = m.launch_count
    invalid = [bgr(frames=0), bgr(frames=capi.MC_MAX_LANES // lanes + 1), bgr(produced=None), bgr(p=None), bgr(info=None),
               bgr(p=bad_mode), bgr(c=2), bgr(in_step=3 * w - 1), bgr(split=3), bgr(canvas=None),
               bgr(canvas=capi.McCanvas(2, c0.data, None, c0.pitch, c0.lane_stride)),
               bgr(canvas=capi.McCanvas(BGR, None, None, c0.pitch, c0.lane_stride)), bgr(canvas=nv_canvas),
               bgr(canvas=capi.McCanvas(BGR, c0.data, None, 3 * cw - 1, c0.lane_stride)),
               bgr(canvas=capi.McCanvas(BGR, c0.data, None, c0.pitch, c0.pitch * chh - 1)),
               nv12(None), nv12(capi.McNv12(nvp.y, None, nvp.pitch, nvp.lane_stride)), nv12(nvp, ww=w - 1),
               nv12(capi.McNv12(nvp.y, nvp.uv, nvp.pitch, nvp.pitch * h - 1)),
               yuv(None), yuv(capi.McYuv422(yst.data, yst.pitch, yst.lane_stride, 2)), yuv(yst, ww=w - 1),
               yuv(capi.McYuv422(yst.data, 2 * w - 1, yst.lane_stride, 0))]
    assert all(st == capi.MC_ERR_INVALID for st in invalid), invalid
    # an overlay of another geometry
    m.set_overlay(synthetic("whole")(cw + 2, chh))
    assert bgr() == capi.MC_ERR_INVALID
    m.clear_overlay()
    # slot buffers that would have to grow while a clip is in flight: a longer clip, and a larger frame
    longer = src.clip(0, n + 1)
    big_cv = Canvas(BGR, cw, chh, (n + 1) * lanes, 2)
    big_buf, big_mc = host_canvas(big_cv, False, lib, keep)
    assert bgr(in_=longer.ctypes.data, frames=n + 1, canvas=big_mc) == capi.MC_ERR_INVALID
    # the device clip calls refuse while compose submits are in flight
    d_in, d_cv = Dev(clips[1]), Canvas(BGR, cw, chh, n * lanes, 2)
    assert lib.mc_chain_compose_device(m._h, d_in.ptr, n, w, h, 3, 3 * w, C.byref(p), 0, LR, C.byref(d_cv.struct()),
                                       ok["produced"], C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert m.launch_count == n0
    # a full pipeline: the second clip is accepted, the third refused
    _, flags1 = src.submit(ch, cfg, clips[1].ctypes.data, n, LR, canvases[1][1])
    n1 = m.launch_count
    assert bgr(in_=clips[2].ctypes.data) == capi.MC_ERR_INVALID and m.launch_count == n1
    for t, fl in enumerate((flags0, flags1)):
        assert m.collect() == bool(want[t][0].any())
        assert np.array_equal(fl, want[t][0]) and np.array_equal(canvases[t][0], want[t][1]), t
        assert np.array_equal(m.lane_produced(), want[t][2]), t
    assert (spare == SENTINEL).all() and (big_buf == SENTINEL).all() and (prod == 0).all()
    for pp in keep:
        lib.mc_host_free(pp)

    # Color's multi-lane refusals, MC_ERR_UNSUPPORTED before anything runs: a held lane, and lanes with other parameters
    color = chain_cfg(O.MODE_COLOR, MODES["color"][1], down=2)
    for refusal in ("hold", "lane_params"):
        cch = L.ProcessingChainB200(0, lanes=lanes)
        if refusal == "hold":
            cch.magnifier.hold_lane(1, True)
        else:
            cch.set_lane_params(1, dataclasses.replace(color.magnification, amplification=7.0))
        n2 = cch.magnifier.launch_count
        ccw, cchh = L.MagnificationProcessor.compose_geometry(color, w, h, 3, NONE)
        ccv = np.full((n * lanes, cchh, 3 * ccw), SENTINEL, np.uint8)
        mc = capi.McCanvas(BGR, ccv.ctypes.data, None, 3 * ccw, 3 * ccw * cchh)
        assert lib.mc_chain_compose_submit(cch.magnifier._h, clips[0].ctypes.data, n, w, h, 3, 3 * w, C.byref(_to_mc(color)), 0,
                                           NONE, C.byref(mc), ok["produced"], C.byref(capi.McChainInfo())) == capi.MC_ERR_UNSUPPORTED
        assert cch.magnifier.launch_count == n2 and (ccv == SENTINEL).all()
        with pytest.raises(capi.MagcoreError):
            cch.collect()   # nothing in flight
        cch.magnifier.close()


def test_errors_return_before_any_launch():
    check_errors(W, H)


# ---- the exporter's shape ----------------------------------------------------------------------------------------------

@pytest.mark.skipif(EMU, reason="1080p clips of 16 on the CPU emulation take too long")
def test_1080p_export_with_labels():
    """1 lane of 1080p BGR, the benchmark's Laplace parameters (6 levels), clips of 16 and a last clip of 7, left/right
    into a BGR canvas with the exporter's labels, pinned, depth 3"""
    w, h, depth, clips = 1920, 1080, 3, (16, 16, 16, 16, 7)
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 6)
    src = ClipSource("bgr", 1, w, h, 0)
    sub, twin = L.ProcessingChainB200(0), L.ProcessingChainB200(0)
    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
    assert (cw, chh) == (2 * w, h)
    ov = export_labels(cw, chh, LR)
    for ch in (sub, twin):
        ch.magnifier.set_overlay(ov)
    base = [lane_frame(t, 0, w, h, 3) for t in range(2)]
    lib, keep, pending = capi.lib(), [], []
    try:
        for i, n in enumerate(clips):
            frames = src.pack([base[(i + t) % 2] for t in range(n)])
            cv = Canvas(BGR, cw, chh, n)
            d_in = Dev(frames)
            tflags, _ = src.device_call(twin.magnifier, cfg, d_in.ptr, n, LR, cv.struct())
            twin.magnifier.sync()
            ref = (tflags.astype(np.uint8), cv.dev.numpy())
            del d_in, cv.dev
            if len(pending) == depth:
                r, canvas, _, flags = pending.pop(0)
                sub.magnifier.collect()
                assert np.array_equal(flags, r[0]) and np.array_equal(canvas, r[1])
            host_in = host_buffer(frames.shape, True, lib, keep, 0)
            host_in[...] = frames
            canvas = host_buffer(ref[1].shape, True, lib, keep, SENTINEL)
            _, flags = src.submit(sub, cfg, host_in.ctypes.data, n, LR, capi.McCanvas(BGR, canvas.ctypes.data, None, 3 * cw, 3 * cw * chh))
            pending.append((ref, canvas, host_in, flags))
        while pending:
            r, canvas, _, flags = pending.pop(0)
            sub.magnifier.collect()
            assert np.array_equal(flags, r[0]) and np.array_equal(canvas, r[1])
        assert r[0].all()
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)
