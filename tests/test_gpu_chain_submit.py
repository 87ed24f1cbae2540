"""The pipelined host chain (mc_chain_submit, mc_chain_submit_nv12, mc_chain_submit_yuv422, collected by mc_collect).

Every case runs a twin handle that calls the device chain (mc_chain_process_device or its _nv12 / _yuv422 form) on device
copies of the same host frames, and must equal it bit for bit: the processed frames and the original tap (padding
included), the flags of every collect, mc_lane_produced after each collect, the info of every submit (magnified 0) and
the state planes at the end.  Restarts, holds, an amplification change, a ROI move and a levels change are submitted
while frames are in flight.  Sentinel bytes show that held lanes, row padding and lanes without a front stage that did
not produce are never written, and mc_lane_produced does not change before a frame is collected.  mc_submit,
mc_submit_nv12 and chain submits interleave on one handle in FIFO order, and every bad submit returns before any launch
with the frames in flight unchanged."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_chain_lanes import MODES, chain_cfg
from test_gpu_lanes import SENTINEL, lane_frame, state_names
from test_gpu_nv12 import Dev, Layout, _pinned, to_nv12
from test_gpu_yuv422 import Yuv, from_bgr

pytestmark = pytest.mark.gpu

EMU = os.environ.get("MC_EMU") == "1"
W, H = 130, 74
ROI, ROI_MOVED = (0.1, 0.15, 0.7, 0.75), (0.2, 0.05, 0.7, 0.75)
FRONTS = {"none": {}, "roi": dict(roi=ROI), "down2": dict(down=2), "down3": dict(down=3), "gray": dict(gray=True),
          "roi_down_gray": dict(roi=ROI, down=2, gray=True)}
SOURCES = ("bgr", "gray", "nv12", "yuyv", "uyvy")
ORDER = {"yuyv": capi.MC_YUV422_YUYV, "uyvy": capi.MC_YUV422_UYVY}


def events_for(lanes, n):
    """{frame: [event]} submitted while frames are in flight: a restart, a hold and its release, an amplification change, a
    ROI move (a structural reset and new tap tables), a levels change"""
    last = lanes - 1
    ev = {3: [("restart", last)], 5: [("hold", min(1, last), 1)], 8: [("hold", min(1, last), 0)], 10: [("amp", 35)],
          13: [("roi", ROI_MOVED)], 16: [("levels", 2)], 18: [("restart", 0)]}
    return {t: e for t, e in ev.items() if t < n}


def apply(chains, cfg, evs, held):
    for e in evs:
        if e[0] == "restart":
            for ch in chains:
                ch.magnifier.restart_lane(e[1])
        elif e[0] == "hold":
            for ch in chains:
                ch.magnifier.hold_lane(e[1], bool(e[2]))
            held[e[1]] = bool(e[2])
        elif e[0] == "amp":
            cfg.magnification.amplification = e[1]
        elif e[0] == "roi":
            cfg.preprocess.roiEnabled = True
            cfg.preprocess.roiX, cfg.preprocess.roiY, cfg.preprocess.roiW, cfg.preprocess.roiH = e[1]
        elif e[0] == "levels":
            cfg.magnification.levels = e[1]


class Source:
    """Frame t of every lane of one source kind as a host buffer with padded rows (and, for NV12, a Cb,Cr plane that does
    not follow the luma plane), and how a call sees it at a given base address."""

    def __init__(self, kind, lanes, w, h, pad):
        self.kind, self.lanes, self.w, self.h = kind, lanes, w, h
        self.c = 1 if kind == "gray" else 3
        self.in_step = w * self.c + pad
        if kind == "nv12":
            self.lay = Layout(w, h, pitch=w + pad, uv_row=h + (4 if pad else 0))
        elif kind in ORDER:
            self.lay = Yuv(w, h, ORDER[kind], pitch=2 * w + pad, lane_rows=2 if pad else 0)

    def frame(self, t):
        lanes, w, h = self.lanes, self.w, self.h
        bgr = [lane_frame(t, k, w, h, 3) for k in range(lanes)]
        if self.kind == "nv12":
            return self.lay.pack(np.stack([to_nv12(f) for f in bgr]), fill=0x3C)
        if self.kind in ORDER:
            return self.lay.pack(np.stack([from_bgr(f, ORDER[self.kind]) for f in bgr]))
        img = np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr]) if self.c == 1 else np.stack(bgr)
        buf = np.full((lanes, h, self.in_step), 0x3C, np.uint8)
        buf[:, :, :w * self.c] = img.reshape(lanes, h, w * self.c)
        return buf

    def device_call(self, ch, cfg, d_in, d_out, out_step, d_orig, orig_step):
        w, h = self.w, self.h
        if self.kind == "nv12":
            return ch.process_nv12_device(self.lay.planes(d_in), 1, w, h, cfg, d_out, out_step, d_orig, orig_step)
        if self.kind in ORDER:
            return ch.process_yuv422_device(self.lay.struct(d_in), 1, w, h, cfg, d_out, out_step, d_orig, orig_step)
        return ch.process_device(d_in, 1, w, h, self.c, self.in_step, cfg, d_out, out_step, d_orig, orig_step)

    def submit(self, ch, cfg, base, out, out_step, orig, orig_step):
        w, h = self.w, self.h
        if self.kind == "nv12":
            return ch.submit_nv12(self.lay.planes(base), w, h, cfg, out, out_step, orig, orig_step)
        if self.kind in ORDER:
            return ch.submit_yuv422(self.lay.struct(base), w, h, cfg, out, out_step, orig, orig_step)
        return ch.submit(base, w, h, self.c, self.in_step, cfg, out, out_step, orig, orig_step)

    def geometry(self, cfg):
        """-> ((rows, row bytes) of out, (rows, row bytes) of original, a front stage runs)"""
        g = L.ProcessingChainB200.geometry(cfg, self.w, self.h, self.c)
        yuv = self.kind in ORDER
        out = (self.h, self.w * self.c) if g.cur_is_input else (g.out_h, g.out_w * g.out_channels)
        orig = (self.h, self.w * self.c) if g.orig_is_input else (g.orig_h, g.orig_w * g.orig_channels)
        return out, orig, yuv or not g.cur_is_input


def host_buffer(shape, pinned, lib, keep, fill):
    a = _pinned(lib, shape, keep) if pinned else np.empty(shape, np.uint8)
    a[...] = fill
    return a


def info_tuple(i):
    return (i.cur_is_input, i.out_w, i.out_h, i.out_channels, i.orig_is_input, i.orig_w, i.orig_h, i.orig_channels, i.magnified)


def check_chain_submit(kind, front, mname, lanes=4, depth=3, pins=(True, False, True), pad=6, n=20, w=W, h=H, events=None,
                       want_orig=True):
    """n frames of `kind` through the chain submits of one handle (pipeline_depth `depth`; pins: whether the input, the
    processed frames and the original tap are pinned) against the twin's device calls."""
    mode, ui = MODES[mname]
    cfg = chain_cfg(mode, ui, **FRONTS[front])
    src = Source(kind, lanes, w, h, pad)
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    if mode == O.MODE_COLOR and lanes > 1:
        for ch in (sub, twin):
            ch.magnifier.set_option("color_lane_lifecycle", 1)
    sub.magnifier.set_option("pipeline_depth", depth)
    evs = events_for(lanes, n) if events is None else events
    lib, keep = capi.lib(), []
    held = [False] * lanes
    ref, pending, collected = [], [], [0]
    last_flags = np.zeros(lanes, bool)

    def collect_one():
        nonlocal last_flags
        assert np.array_equal(sub.magnifier.lane_produced(), last_flags)   # unchanged until the frame is collected
        i = collected[0]
        flags = sub.collect()
        r, (out, orig, _) = ref[i], pending.pop(0)
        assert np.array_equal(flags, r["flags"]), i
        assert np.array_equal(sub.magnifier.lane_produced(), r["lane_produced"]), i
        assert np.array_equal(out, r["out"]), (i, np.argwhere(out != r["out"])[:5])
        if orig is not None:
            assert np.array_equal(orig, r["orig"]), i
            assert (orig[:, :, r["orig_row"]:] == SENTINEL).all(), i
        assert (out[:, :, r["out_row"]:] == SENTINEL).all(), i                      # row padding
        for k in range(lanes):
            if r["held"][k]:
                assert (out[k] == SENTINEL).all() and (orig is None or (orig[k] == SENTINEL).all()), (i, k)
            elif not r["front"] and not flags[k]:
                assert (out[k] == SENTINEL).all(), (i, k)                           # the input is the result
        last_flags = flags
        collected[0] += 1

    try:
        for t in range(n):
            apply((sub, twin), cfg, evs.get(t, []), held)
            (oh, orow), (gh, grow), front_runs = src.geometry(cfg)
            ostep, gstep = orow + pad, grow + pad
            frame = src.frame(t)
            d_in = Dev(frame)
            d_out = Dev(np.full((lanes, oh, ostep), SENTINEL, np.uint8))
            d_orig = Dev(np.full((lanes, gh, gstep), SENTINEL, np.uint8)) if want_orig else None
            flags, tinfo = src.device_call(twin, cfg, d_in.ptr, d_out.ptr, ostep, d_orig.ptr if d_orig else 0, gstep)
            twin.magnifier.sync()
            ref.append(dict(flags=flags[0], lane_produced=twin.magnifier.lane_produced(), out=d_out.numpy(),
                            orig=d_orig.numpy() if d_orig else None, out_row=orow, orig_row=grow, held=list(held),
                            front=front_runs))
            if len(pending) == depth:
                collect_one()
            host_in = host_buffer(frame.shape, pins[0], lib, keep, 0)
            host_in[...] = frame
            out = host_buffer((lanes, oh, ostep), pins[1], lib, keep, SENTINEL)
            orig = host_buffer((lanes, gh, gstep), pins[2], lib, keep, SENTINEL) if want_orig else None
            pending.append((out, orig, host_in))   # every buffer stays valid until its frame is collected
            info = src.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, ostep, orig.ctypes.data if want_orig else 0, gstep)
            assert info_tuple(info) == info_tuple(tinfo)[:-1] + (0,), t
        while pending:
            collect_one()
        for name, level in state_names(twin.magnifier, mode):
            assert np.array_equal(sub.magnifier.get_state(name, level), twin.magnifier.get_state(name, level)), (name, level)
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)


# ---- sources x fronts ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("front", list(FRONTS))
@pytest.mark.parametrize("kind", SOURCES)
def test_sources_and_fronts_equal_the_device_chain(kind, front):
    i = SOURCES.index(kind) + list(FRONTS).index(front)
    pins = [(True, True, True), (False, False, False), (True, False, True), (False, True, False)][i % 4]
    check_chain_submit(kind, front, "laplace", lanes=4, depth=3, pins=pins)


# ---- modes x lanes x pipeline depths ----------------------------------------------------------------------------------

@pytest.mark.parametrize("depth", [1, 3, 5])
@pytest.mark.parametrize("lanes", [1, 4])
@pytest.mark.parametrize("mname", ["laplace", "phase", "color"])
def test_modes_lanes_and_depths(mname, lanes, depth):
    kind = ["bgr", "yuyv", "nv12"][depth // 2]
    front = "roi_down_gray" if depth != 3 else "down2"
    check_chain_submit(kind, front, mname, lanes=lanes, depth=depth, pins=(depth == 1, depth != 1, lanes == 1), n=24)


@pytest.mark.parametrize("pins", [(False, False, False), (True, False, False), (False, True, True), (True, True, False)],
                         ids=["pageable", "pinned_in", "pinned_out", "pinned_in_out"])
@pytest.mark.parametrize("pad", [0, 6], ids=["tight", "padded"])
def test_pinned_and_pageable_buffers(pins, pad):
    check_chain_submit("nv12", "roi", "phase", lanes=3, depth=3, pins=pins, pad=pad)


def test_no_original_buffer():
    check_chain_submit("yuyv", "down3", "laplace", lanes=2, want_orig=False)


# ---- FIFO across every submit of one handle ----------------------------------------------------------------------------

def check_interleaved(w, h, lanes=2, n=12, pinned=False):
    """mc_submit, mc_submit_nv12, mc_chain_submit and mc_chain_submit_yuv422 in turn on one handle: each collected frame
    equals its own call on a twin handle that runs the device calls in the same order"""
    mode, ui = MODES["laplace"]
    cfg = chain_cfg(mode, ui)   # one geometry: the calls share the temporal state without a structural reset
    plain = cfg
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    lay = Layout(w, h, pitch=w + 2)
    srcs = {"bgr": Source("bgr", lanes, w, h, 4), "yuyv": Source("yuyv", lanes, w, h, 4)}
    lib, keep, pending, ref = capi.lib(), [], [], []
    try:
        for t in range(n):
            which = ("chain_yuyv", "submit", "submit_nv12", "chain_bgr")[t % 4]
            if which == "submit":
                x = np.stack([lane_frame(t, k, w, h, 3) for k in range(lanes)])
                d_in, d_out = Dev(x), Dev(np.full_like(x, SENTINEL))
                prod = twin.magnifier.process_device(d_in.ptr, w, h, 3, 3 * w, plain, d_out.ptr, 3 * w)
                host_in, out = host_buffer(x.shape, pinned, lib, keep, 0), host_buffer(x.shape, pinned, lib, keep, SENTINEL)
                host_in[...] = x
                sub.magnifier.submit(host_in.ctypes.data, w, h, 3, 3 * w, plain, out.ctypes.data, 3 * w)
                outs = (out,)
            elif which == "submit_nv12":
                x = lay.pack(np.stack([to_nv12(lane_frame(t, k, w, h, 3)) for k in range(lanes)]))
                d_in, d_out = Dev(x), Dev(np.full_like(x, SENTINEL))
                prod = twin.magnifier.process_nv12_device(lay.planes(d_in.ptr), w, h, plain, lay.planes(d_out.ptr))
                host_in, out = host_buffer(x.shape, pinned, lib, keep, 0), host_buffer(x.shape, pinned, lib, keep, SENTINEL)
                host_in[...] = x
                sub.magnifier.submit_nv12(lay.planes(host_in.ctypes.data), w, h, plain, lay.planes(out.ctypes.data))
                outs = (out,)
            else:
                src = srcs[which[6:]]
                frame = src.frame(t)
                (oh, orow), (gh, grow), _ = src.geometry(cfg)
                d_in, d_out, d_orig = Dev(frame), Dev(np.full((lanes, oh, orow), SENTINEL, np.uint8)), Dev(
                    np.full((lanes, gh, grow), SENTINEL, np.uint8))
                flags, _ = src.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
                prod = bool(flags.any())
                host_in = host_buffer(frame.shape, pinned, lib, keep, 0)
                host_in[...] = frame
                out = host_buffer((lanes, oh, orow), pinned, lib, keep, SENTINEL)
                orig = host_buffer((lanes, gh, grow), pinned, lib, keep, SENTINEL)
                src.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, orow, orig.ctypes.data, grow)
                outs = (out, orig)
                d_out = (d_out, d_orig)
            twin.magnifier.sync()
            want = tuple(d.numpy() for d in (d_out if isinstance(d_out, tuple) else (d_out,)))
            ref.append((which, prod, twin.magnifier.lane_produced(), want))
            pending.append((outs, host_in))
            if len(pending) == 3 or t < 2:   # the slots grow to the 4:2:2 output and the BGR input while nothing is in flight
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
    which, prod, lane_prod, want = ref[i]
    outs, _ = pending.pop(0)
    assert sub.magnifier.collect() == prod, (i, which)
    assert np.array_equal(sub.magnifier.lane_produced(), lane_prod), (i, which)
    for got, exp in zip(outs, want):
        assert np.array_equal(got, exp), (i, which)


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_every_submit_interleaves_in_fifo_order(pinned):
    check_interleaved(W, H, pinned=pinned)


# ---- errors --------------------------------------------------------------------------------------------------------------

def check_errors(w, h, lanes=2):
    """Every bad submit returns its code with the launch count unchanged; the next mc_collect still returns the frame
    submitted before it.  The device chain calls refuse while chain frames are in flight."""
    mode, ui = MODES["laplace"]
    cfg = chain_cfg(mode, ui, down=2, roi=ROI, gray=True)
    lib, p = capi.lib(), _to_mc(cfg)
    ch, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    ch.magnifier.set_option("pipeline_depth", 2)
    m = ch.magnifier
    src = Source("bgr", lanes, w, h, 0)
    nv = Source("nv12", lanes, w, h, 4)
    yv = Source("yuyv", lanes, w, h, 4)
    (oh, orow), (gh, grow), _ = src.geometry(cfg)
    frames = [src.frame(t) for t in range(3)]
    outs = [np.full((lanes, oh, orow), SENTINEL, np.uint8) for _ in range(3)]
    origs = [np.full((lanes, gh, grow), SENTINEL, np.uint8) for _ in range(3)]
    want = []
    for t in range(2):
        d_in, d_out, d_orig = Dev(frames[t]), Dev(outs[t]), Dev(origs[t])
        src.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
        twin.magnifier.sync()
        want.append((d_out.numpy(), d_orig.numpy(), twin.magnifier.lane_produced()))
    src.submit(ch, cfg, frames[0].ctypes.data, outs[0].ctypes.data, orow, origs[0].ctypes.data, grow)
    nvf, yvf = nv.frame(0), yv.frame(0)
    nvp, yvs = nv.lay.planes(nvf.ctypes.data), yv.lay.struct(yvf.ctypes.data)
    spare_out, spare_orig = np.full_like(outs[0], SENTINEL), np.full_like(origs[0], SENTINEL)
    ok = dict(in_=frames[1].ctypes.data, w=w, h=h, c=3, in_step=3 * w, p=p, gray=1, out=spare_out.ctypes.data, out_step=orow,
              orig=spare_orig.ctypes.data, orig_step=grow)

    def bgr(**kw):
        a = {**ok, **kw}
        return lib.mc_chain_submit(m._h, a["in_"], a["w"], a["h"], a["c"], a["in_step"], a["p"] and C.byref(a["p"]), a["gray"],
                                   a["out"], a["out_step"], a["orig"], a["orig_step"], C.byref(capi.McChainInfo()))

    def nv12(planes, ww=w, hh=h, out=ok["out"]):
        return lib.mc_chain_submit_nv12(m._h, planes and C.byref(planes), ww, hh, C.byref(p), 1, out, orow, ok["orig"], grow,
                                        C.byref(capi.McChainInfo()))

    def yuv(frame, ww=w, hh=h):
        return lib.mc_chain_submit_yuv422(m._h, frame and C.byref(frame), ww, hh, C.byref(p), 1, ok["out"], orow, ok["orig"],
                                          grow, C.byref(capi.McChainInfo()))

    bad_mode = _to_mc(cfg)
    bad_mode.mode = 7
    n0 = m.launch_count
    invalid = [bgr(in_step=3 * w - 1), bgr(out_step=orow - 1), bgr(orig_step=grow - 1), bgr(out=None), bgr(c=2), bgr(p=None),
               bgr(p=bad_mode),
               nv12(None), nv12(capi.McNv12(nvp.y, None, nvp.pitch, nvp.lane_stride)), nv12(nvp, ww=w - 1),
               nv12(capi.McNv12(nvp.y, nvp.uv, w - 1, nvp.lane_stride)), nv12(capi.McNv12(nvp.y, nvp.uv, nvp.pitch, nvp.pitch * h - 1)),
               nv12(nvp, out=None),
               yuv(None), yuv(capi.McYuv422(None, yvs.pitch, yvs.lane_stride, 0)), yuv(capi.McYuv422(yvs.data, yvs.pitch, yvs.lane_stride, 2)),
               yuv(yvs, ww=w - 1), yuv(capi.McYuv422(yvs.data, 2 * w - 1, yvs.lane_stride, 0)),
               yuv(capi.McYuv422(yvs.data, yvs.pitch, yvs.pitch * h - 1, 0))]
    assert all(st == capi.MC_ERR_INVALID for st in invalid), invalid
    # slot buffers that would have to grow while a frame is in flight
    big = np.zeros((lanes, 2 * h, 2 * w * 3), np.uint8)
    assert lib.mc_chain_submit(m._h, big.ctypes.data, 2 * w, 2 * h, 3, 6 * w, C.byref(p), 1, big.ctypes.data, 6 * w, None, 0,
                               C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    # the device chain calls refuse while chain frames are in flight
    d_in, d_out = Dev(frames[1]), Dev(outs[2])
    flags = np.zeros(lanes, np.uint8)
    assert lib.mc_chain_process_device(m._h, d_in.ptr, 1, w, h, 3, 3 * w, C.byref(p), 1, d_out.ptr, orow, None, 0,
                                       flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert m.launch_count == n0
    # a full pipeline: the second frame is accepted, the third refused
    src.submit(ch, cfg, frames[1].ctypes.data, outs[1].ctypes.data, orow, origs[1].ctypes.data, grow)
    n1 = m.launch_count
    assert bgr(in_=frames[2].ctypes.data) == capi.MC_ERR_INVALID and m.launch_count == n1
    for t in range(2):
        ch.collect()
        assert np.array_equal(outs[t], want[t][0]) and np.array_equal(origs[t], want[t][1]), t
        assert np.array_equal(m.lane_produced(), want[t][2]), t
    assert (spare_out == SENTINEL).all() and (spare_orig == SENTINEL).all()

    # Color's multi-lane refusal with a held lane: MC_ERR_UNSUPPORTED before anything runs
    color = chain_cfg(O.MODE_COLOR, MODES["color"][1], down=2, gray=True)
    cch = L.ProcessingChainB200(0, lanes=lanes)
    cch.magnifier.hold_lane(1, True)
    n2 = cch.magnifier.launch_count
    (coh, corow), _, _ = src.geometry(color)
    color_out = np.full((lanes, coh, corow), SENTINEL, np.uint8)
    assert lib.mc_chain_submit(cch.magnifier._h, frames[0].ctypes.data, w, h, 3, 3 * w, C.byref(_to_mc(color)), 1,
                               color_out.ctypes.data, corow, None, 0, C.byref(capi.McChainInfo())) == capi.MC_ERR_UNSUPPORTED
    assert cch.magnifier.launch_count == n2
    with pytest.raises(capi.MagcoreError):
        cch.collect()   # nothing in flight


def test_errors_return_before_any_launch():
    check_errors(W, H)


# ---- a user-sized case ---------------------------------------------------------------------------------------------------

@pytest.mark.skipif(EMU, reason="16 lanes of 1080p on the CPU emulation take too long")
def test_16_lanes_of_1080p_yuyv():
    """16 lanes of 1080p YUYV, downscale 2, the benchmark's Laplace parameters (6 levels), pinned, depth 3"""
    lanes, w, h, n, depth = 16, 1920, 1080, 6, 3
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 6)
    cfg.preprocess = L.PreprocessParams(2)
    src = Source("yuyv", lanes, w, h, 0)
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    (oh, orow), (gh, grow), _ = src.geometry(cfg)
    lib, keep = capi.lib(), []
    base = [src.frame(t) for t in range(2)]
    try:
        pending, ref = [], []
        for t in range(n):
            frame = base[t % 2]
            d_in, d_out, d_orig = Dev(frame), Dev(np.zeros((lanes, oh, orow), np.uint8)), Dev(np.zeros((lanes, gh, grow), np.uint8))
            flags, _ = src.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
            twin.magnifier.sync()
            ref.append((flags[0], d_out.numpy(), d_orig.numpy()))
            del d_in, d_out, d_orig
            if len(pending) == depth:
                out, orig = pending.pop(0)
                i = t - depth
                assert np.array_equal(sub.collect(), ref[i][0]) and np.array_equal(out, ref[i][1]) and np.array_equal(orig, ref[i][2]), i
            host_in = host_buffer(frame.shape, True, lib, keep, 0)
            host_in[...] = frame
            out, orig = host_buffer((lanes, oh, orow), True, lib, keep, 0), host_buffer((lanes, gh, grow), True, lib, keep, 0)
            src.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, orow, orig.ctypes.data, grow)
            pending.append((out, orig))
        for i in range(n - depth, n):
            out, orig = pending.pop(0)
            assert np.array_equal(sub.collect(), ref[i][0]) and np.array_equal(out, ref[i][1]) and np.array_equal(orig, ref[i][2]), i
        assert ref[-1][0].all()
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)
