"""Packed 4:2:2 camera frames (YUYV / UYVY) into the processing chain: mc_chain_process_yuv422_device,
mc_chain_compose_yuv422_device and the blocking host call mc_chain_process_yuv422.

For any 4:2:2 input X a call must equal the BGR chain call on B = cv2.cvtColor(X, COLOR_YUV2BGR_YUYV / _UYVY), bit for
bit: flags, lane flags, processed frames, original tap and state.  The conversion counts as a front stage that always
runs, so where the BGR call leaves its result to the input, the 4:2:2 call writes B (or its gray) and reports both
*_is_input flags as 0.  A twin handle takes the BGR calls on cv2's conversion; every buffer is sentinel-filled, padding
included, so bytes written where they should not be show up."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from compose_oracle import compose
from test_gpu_chain_lanes import MODES, chain_cfg, device_call, info_tuple, none_cfg, out_geom
from test_gpu_compose import SPLITS, Canvas, image
from test_gpu_lanes import SENTINEL, lane_frame, state_names
from test_gpu_nv12 import Dev, Layout, composition, to_bgr, to_nv12

EMU = os.environ.get("MC_EMU") == "1"
ORDERS = {"yuyv": capi.MC_YUV422_YUYV, "uyvy": capi.MC_YUV422_UYVY}
CODES = {capi.MC_YUV422_YUYV: cv2.COLOR_YUV2BGR_YUYV, capi.MC_YUV422_UYVY: cv2.COLOR_YUV2BGR_UYVY}


# ---- 4:2:2 frames, as a camera delivers them ------------------------------------------------------------------------

def from_bgr(bgr, order):
    """BGR [h][w][3] -> a packed 4:2:2 frame [h][2w] of that order: each pixel's luma and its pair's left chroma (any bytes
    are a valid input; this keeps the synthetic motion visible)"""
    ycc = cv2.cvtColor(bgr, cv2.COLOR_BGR2YCrCb)
    h, w = bgr.shape[:2]
    y, cr, cb = ycc[..., 0].reshape(h, w // 2, 2), ycc[:, ::2, 1], ycc[:, ::2, 2]
    grp = [y[..., 0], cb, y[..., 1], cr] if order == capi.MC_YUV422_YUYV else [cb, y[..., 0], cr, y[..., 1]]
    return np.stack(grp, -1).reshape(h, 2 * w)


def convert(x, order):
    """cv2's conversion of packed frames [..][h][2w] -> BGR [..][h][w][3]"""
    h, w2 = x.shape[-2:]
    flat = x.reshape(-1, h, w2)
    return np.stack([cv2.cvtColor(np.ascontiguousarray(f).reshape(h, w2 // 2, 2), CODES[order]) for f in flat]).reshape(
        x.shape[:-2] + (h, w2 // 2, 3))


class Yuv:
    """Where frame set's frames sit: lanes blocks of h + lane_rows rows of `pitch` bytes (>= 2w), `offset` bytes from
    the buffer's start."""

    def __init__(self, w, h, order, pitch=None, lane_rows=0, offset=0):
        self.w, self.h, self.order = w, h, order
        self.pitch = pitch or 2 * w
        self.rows = h + lane_rows
        self.offset = offset

    @property
    def lane_stride(self):
        return self.pitch * self.rows

    def pack(self, x, fill=0x3C):
        buf = np.full(len(x) * self.lane_stride + self.offset, fill, np.uint8)
        view = buf[self.offset:].reshape(len(x), self.rows, self.pitch)
        view[:, :self.h, :2 * self.w] = x
        return buf

    def struct(self, base, **override):
        f = dict(data=base + self.offset, pitch=self.pitch, lane_stride=self.lane_stride, order=self.order)
        f.update(override)
        return capi.McYuv422(f["data"], f["pitch"], f["lane_stride"], f["order"])


def yuv_info(binfo, w, h, gray):
    """the info a 4:2:2 call reports, from the BGR call's: both frames are written"""
    ow, oh = (w, h) if binfo.cur_is_input and binfo.orig_is_input else (
        (binfo.orig_w, binfo.orig_h) if not binfo.orig_is_input else (binfo.out_w, binfo.out_h))
    return (0, ow, oh, 1 if gray else 3, 0, ow, oh, 3, binfo.magnified)


def yuv_device_call(ch, cfg, x, frames, lay, out_pad=0, orig_pad=0, want_orig=True):
    """one mc_chain_process_yuv422_device call on packed frames x [V][h][2w] -> (flags, info, out, orig)"""
    g = ch.geometry(cfg, lay.w, lay.h, 3)
    dw, dh = (lay.w, lay.h) if g.cur_is_input and g.orig_is_input else (
        (g.orig_w, g.orig_h) if not g.orig_is_input else (g.out_w, g.out_h))
    cc = 1 if cfg.grayscale else 3
    v = len(x)
    out_step, orig_step = dw * cc + out_pad, dw * 3 + orig_pad
    d_in = Dev(lay.pack(x))
    d_out = Dev(np.full((v, dh, out_step), SENTINEL, np.uint8))
    d_orig = Dev(np.full((v, dh, orig_step), SENTINEL, np.uint8)) if want_orig else None
    flags, info = ch.process_yuv422_device(lay.struct(d_in.ptr), frames, lay.w, lay.h, cfg, d_out.ptr, out_step,
                                           d_orig.ptr if d_orig else 0, orig_step)
    ch.magnifier.sync()
    return flags.astype(np.uint8), info, d_out.numpy(), d_orig.numpy() if d_orig else None


def filled(buf, row, images):
    """sentinel-filled copy of buf's shape with images[v] (None: untouched) in the first `row` bytes of its rows"""
    want = np.full(buf.shape, SENTINEL, np.uint8)
    for v, im in enumerate(images):
        if im is not None:
            want[v, :, :row] = im.reshape(buf.shape[1], row)
    return want


# ---- the chain against the BGR chain on cv2's conversion --------------------------------------------------------------

def check_yuv(mode, ui, w, h, steps, lanes=1, lay_kw=None, order=capi.MC_YUV422_YUYV, launches=True, want_orig=True,
              pads=(0, 0)):
    """Handle A takes 4:2:2 calls, its twin B the BGR chain calls (mc_chain_process_device) on cv2's conversion of the same
    frames.  steps: ("frame",) / ("clip", n) calls; ("bgr",) / ("nv12",) that call on both (A and B must agree);
    ("restart", k) / ("hold", k, on) on both; ("cfg", kwargs) chain settings (down / roi / gray).  After every 4:2:2 call
    A's flags, lane flags and info are B's (both frames written), d_out is B's where B wrote it and B's input or its
    gray elsewhere, d_original B's tap or B's input; held lanes stay untouched.  At the end the state planes are equal."""
    cfg = chain_cfg(mode, ui)
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    if launches:
        for ch in (a, b):
            ch.magnifier.set_option("profile_kernels", 1)
    lay = Yuv(w, h, order, **(lay_kw or {}))
    held, t = [False] * lanes, 0
    for step in steps:
        if step[0] in ("restart", "hold"):
            for ch in (a, b):
                ch.magnifier.restart_lane(step[1]) if step[0] == "restart" else ch.magnifier.hold_lane(step[1], step[2])
            if step[0] == "hold":
                held[step[1]] = bool(step[2])
            continue
        if step[0] == "cfg":
            cfg = chain_cfg(mode, ui, **step[1])
            continue
        n = step[1] if step[0] == "clip" else 1
        bgr = np.stack([lane_frame(s, k, w, h, 3) for s in range(t, t + n) for k in range(lanes)])
        t += n
        if step[0] in ("bgr", "nv12"):
            nv = Layout(w, h) if step[0] == "nv12" else None
            src = np.stack([to_nv12(f) for f in bgr]) if nv else bgr
            ra = device_call(a, cfg, src, n, w, h, 3, nv12=nv)
            rb = device_call(b, cfg, np.stack([to_bgr(f) for f in src]) if nv else bgr, n, w, h, 3)
            assert np.array_equal(ra[0], rb[0]) and info_tuple(ra[1]) == info_tuple(rb[1]), step
            assert np.array_equal(ra[2], rb[2]) and np.array_equal(ra[3], rb[3]), step
            continue
        x = np.stack([from_bgr(f, order) for f in bgr])
        seen = convert(x, order)
        if launches:
            a.magnifier.profile_read()
            b.magnifier.profile_read()
        flags, info, out, orig = yuv_device_call(a, cfg, x, n, lay, *pads, want_orig=want_orig)
        bflags, binfo, bout, borig = device_call(b, cfg, seen, n, w, h, 3)
        assert np.array_equal(flags, bflags), (step, flags, bflags)
        assert info_tuple(info) == yuv_info(binfo, w, h, cfg.grayscale), (step, info_tuple(info), info_tuple(binfo))
        assert np.array_equal(a.magnifier.lane_produced(), b.magnifier.lane_produced())
        (orows, _), (grows, _) = out_geom(b, cfg, w, h, 3)
        row = info.out_w * info.out_channels
        outs, origs = [], []
        for v in range(n * lanes):
            if held[v % lanes]:
                outs.append(None)
                origs.append(None)
                continue
            if binfo.cur_is_input and not bflags.ravel()[v]:
                outs.append(seen[v])
            else:
                outs.append(image(bout[v], orows, info.out_w, info.out_channels))
            origs.append(seen[v] if binfo.orig_is_input else image(borig[v], grows, info.orig_w, 3))
        assert np.array_equal(out, filled(out, row, outs)), step
        if want_orig:
            assert np.array_equal(orig, filled(orig, info.orig_w * 3, origs)), step
        if launches:
            ca, cb = composition(a.magnifier), composition(b.magnifier)
            cb[("chain_front", 0)] = 1
            assert ca == cb, (step, ca, cb)
    for n_, l in (state_names(b.magnifier, mode) if mode != O.MODE_NONE else []):
        assert np.array_equal(a.magnifier.get_state(n_, l), b.magnifier.get_state(n_, l)), (n_, l)
    return a


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu

W, H = (66, 37) if EMU else (130, 75)   # odd height


def every_triple(order, w, h):
    """-> a packed frame [h][2w] whose first 2^23 groups (when w * h >= 2^24) hold every (Y, Cb, Cr) triple once"""
    i = np.arange(w * h // 2, dtype=np.uint32) % (1 << 23)
    y0, u, v = (i >> 16) * 2, (i >> 8) & 255, i & 255
    grp = [y0, u, y0 + 1, v] if order == capi.MC_YUV422_YUYV else [u, y0, v, y0 + 1]
    return np.stack(grp, -1).astype(np.uint8).reshape(h, 2 * w)


@pytest.mark.skipif(EMU, reason="every triple is too slow for the CPU emulation")
@pytest.mark.parametrize("order", list(ORDERS))
@pytest.mark.parametrize("w,h,pitch_pad", [(4096, 4096, 0), (4096, 4095, 2), (4090, 4096, 64), (4090, 4093, 1)])
def test_front_on_every_triple(order, w, h, pitch_pad):
    """Mode None, no Preprocess stage: d_original is cv2's conversion and d_out its gray, over a 4096 x 4096 frame that
    holds every triple; pitches 2w (32-bit groups), 2w + 2 (bytes), 2w + 64, and an odd one; width = 2 mod 8; odd heights"""
    o = ORDERS[order]
    x = every_triple(o, w, h)
    want = convert(x[None], o)[0]
    ch = L.ProcessingChainB200(0)
    flags, info, out, orig = yuv_device_call(ch, none_cfg(gray=True), x[None], 1, Yuv(w, h, o, pitch=2 * w + pitch_pad))
    assert not flags.any() and info_tuple(info) == (0, w, h, 1, 0, w, h, 3, 0)
    assert np.array_equal(orig[0], want.reshape(h, 3 * w))
    assert np.array_equal(out[0], cv2.cvtColor(want, cv2.COLOR_BGR2GRAY))


FRONT_CASES = [
    # (down, roi, gray)
    (1, None, False), (1, None, True), (2, None, False), (3, None, True), (4, (0.1, 0.2, 0.77, 0.61), True),
    (1, (0.015, 0.0, 0.5, 1.0), False),    # crop at an odd column: pixels pair with their frame neighbours
    (3, (0.1, 0.15, 0.8, 0.75), False),    # fractional INTER_AREA
    (2, (0.997, 0.995, 0.5, 0.5), True),   # 1 x 1 output
]


@pytest.mark.parametrize("order", list(ORDERS))
@pytest.mark.parametrize("down,roi,gray", FRONT_CASES)
def test_front_matches_the_bgr_front(order, down, roi, gray):
    """Mode None over 3 lanes x 2 frames with padded rows and an unaligned start (byte path)"""
    check_yuv(O.MODE_NONE, MODES["laplace"][1], W, H, [("cfg", dict(down=down, roi=roi, gray=gray)), ("clip", 2)], lanes=3,
              order=ORDERS[order], lay_kw=dict(pitch=2 * W + 6, lane_rows=1, offset=1), pads=(3, 5))


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("settings", [dict(), dict(gray=True), dict(down=2), dict(down=3, roi=(0.05, 0.1, 0.9, 0.85)),
                                      dict(down=2, gray=True)], ids=["none", "gray", "down2", "roi_down3", "down2_gray"])
@pytest.mark.parametrize("lanes", [1, 3])
def test_chain_equals_bgr_chain_on_cv2_conversion(mname, settings, lanes):
    """frames and clips (T = 1, 4), restart and hold (not Color, which refuses them across lanes), UYVY on 3 lanes"""
    mode, ui = MODES[mname]
    lifecycle = [] if mname == "color" or lanes == 1 else [("restart", 2), ("hold", 1, 1), ("frame",), ("clip", 2),
                                                            ("hold", 1, 0)]
    steps = [("cfg", settings), ("frame",), ("frame",), ("clip", 4), *lifecycle, ("frame",), ("clip", 1)]
    order = capi.MC_YUV422_UYVY if lanes == 3 else capi.MC_YUV422_YUYV
    check_yuv(mode, ui, W, H, steps, lanes=lanes, order=order, lay_kw=dict(pitch=2 * W + 64))


@pytest.mark.parametrize("mname", list(MODES))
def test_yuv422_nv12_and_bgr_calls_interleave(mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("bgr",), ("frame",), ("nv12",), ("clip", 3), ("bgr",), ("nv12",), ("frame",),
             ("cfg", dict(down=2)), ("frame",), ("nv12",), ("frame",)]
    check_yuv(mode, ui, W, H + H % 2, steps, lanes=2)   # NV12 needs an even height


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_no_original_buffer(mname):
    """d_original NULL: the front stages B as the magnifier's input; d_out is still written for every lane"""
    mode, ui = MODES[mname]
    check_yuv(mode, ui, W, H, [("frame",), ("clip", 3), ("cfg", dict(gray=True)), ("frame",)], lanes=2, want_orig=False)


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
@pytest.mark.parametrize("mname", list(MODES))
def test_1080p(mname):
    mode, ui = MODES[mname]
    check_yuv(mode, ui, 1920, 1080, [("frame",), ("frame",), ("clip", 3), ("frame",)], lanes=1,
              lay_kw=dict(pitch=3840))


# ---- compose -------------------------------------------------------------------------------------------------------

def check_compose_yuv(mode, ui, w, h, fmt, split, steps, lanes=1, gray=False, order=capi.MC_YUV422_YUYV, lay_kw=None,
                      pad=0, lane_rows=0, uv_gap=0):
    """Handle A takes compose calls on 4:2:2 frames, its twin B the BGR chain calls on cv2's conversion: A's canvas is
    compose() of B's taps with B's input standing where B leaves the result to the input."""
    cfg = chain_cfg(mode, ui, gray=gray)
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    lay = Yuv(w, h, order, **(lay_kw or {}))
    held, t = [False] * lanes, 0
    for step in steps:
        if step[0] in ("restart", "hold"):
            for ch in (a, b):
                ch.magnifier.restart_lane(step[1]) if step[0] == "restart" else ch.magnifier.hold_lane(step[1], step[2])
            if step[0] == "hold":
                held[step[1]] = bool(step[2])
            continue
        if step[0] == "cfg":
            cfg = chain_cfg(mode, ui, gray=gray, **step[1])
            continue
        n = step[1] if step[0] == "clip" else 1
        bgr = np.stack([lane_frame(s, k, w, h, 3) for s in range(t, t + n) for k in range(lanes)])
        t += n
        x = np.stack([from_bgr(f, order) for f in bgr])
        seen = convert(x, order)
        v = n * lanes
        cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, split)
        cv = Canvas(fmt, cw, chh, v, pad, lane_rows, uv_gap)
        d_in = Dev(lay.pack(x))
        flags, info = a.magnifier.chain_compose_yuv422_device(lay.struct(d_in.ptr), n, w, h, cfg, split, cv.struct())
        a.magnifier.sync()
        bflags, binfo, out, orig = device_call(b, cfg, seen, n, w, h, 3)
        assert np.array_equal(flags.astype(np.uint8), bflags), step
        assert info_tuple(info) == yuv_info(binfo, w, h, gray), (step, info_tuple(info))
        (orows, _), (grows, _) = out_geom(b, cfg, w, h, 3)
        cur_dims = (w, 3) if binfo.cur_is_input else (binfo.out_w, binfo.out_channels)
        canvases = []
        for k in range(v):
            if held[k % lanes]:
                canvases.append(None)
                continue
            cur = seen[k] if binfo.cur_is_input and not bflags.ravel()[k] else image(out[k], orows, *cur_dims)
            original = seen[k] if binfo.orig_is_input else image(orig[k], grows, binfo.orig_w, 3)
            canvases.append(compose(original, cur, split))
        assert np.array_equal(cv.dev.numpy(), cv.expected(canvases)), step
    for n_, l in state_names(b.magnifier, mode):
        assert np.array_equal(a.magnifier.get_state(n_, l), b.magnifier.get_state(n_, l)), (n_, l)


@pytest.mark.parametrize("fmt", [capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12], ids=["bgr_canvas", "nv12_canvas"])
@pytest.mark.parametrize("gray", [False, True], ids=["color", "grayscale"])
@pytest.mark.parametrize("split", list(SPLITS))
@pytest.mark.parametrize("order", list(ORDERS))
def test_compose_splits_and_canvases(order, split, gray, fmt):
    steps = [("frame",), ("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 3), ("cfg", dict(down=2)),
             ("frame",), ("cfg", dict()), ("clip", 2)]
    check_compose_yuv(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, SPLITS[split], steps, lanes=2, gray=gray,
                      order=ORDERS[order], pad=5, lane_rows=1, uv_gap=3)


@pytest.mark.parametrize("mname", ["phase", "color"])
@pytest.mark.parametrize("aligned", [True, False])
def test_compose_frames_not_produced_and_lanes(mname, aligned):
    """Phase's first frame and Color's warm-up show B; aligned 64-bit pane reads or the byte path; a hold on 3 lanes"""
    mode, ui = MODES[mname]
    lanes = 1 if mname == "color" else 3
    hold = [("hold", 1, 1), ("clip", 2), ("hold", 1, 0)] if lanes > 1 else []
    lay_kw = dict(pitch=2 * 64) if aligned else dict(pitch=2 * 64 + 2, offset=2)
    check_compose_yuv(mode, ui, 64, 32, capi.MC_CANVAS_NV12, capi.MC_SPLIT_LEFT_RIGHT, [("frame",), ("clip", 3), *hold, ("frame",)],
                      lanes=lanes, gray=not aligned, lay_kw=lay_kw)


# ---- the blocking host call --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("settings", [dict(), dict(down=2, gray=True)], ids=["none", "down2_gray"])
@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_host_call_equals_bgr_run_chain_once(mname, settings, pinned):
    """mc_chain_process_yuv422 on a padded host frame (pinned or pageable) against run_chain_once on cv2's conversion;
    the Python run_chain_once of a "YUYV" Frame gives the same"""
    mode, ui = MODES[mname]
    cfg = chain_cfg(mode, ui, **settings)
    w, h, pitch = W, H, 2 * W + 10
    lib, keep = capi.lib(), []
    a, b, c = (L.ProcessingChainB200(0) for _ in range(3))
    try:
        for t in range(4):
            x = from_bgr(lane_frame(t, 0, w, h, 3), capi.MC_YUV422_YUYV)
            seen = convert(x, capi.MC_YUV422_YUYV)
            buf = np.full((h, pitch), 0x3C, np.uint8)
            buf[:, :2 * w] = x
            if pinned:
                p = lib.mc_host_alloc(buf.size)
                keep.append(p)
                host = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=buf.shape)
                host[...] = buf
            else:
                host = buf
            g = b.geometry(cfg, w, h, 3)
            dw, dh = (w, h) if g.orig_is_input and g.cur_is_input else ((g.orig_w, g.orig_h) if not g.orig_is_input else (g.out_w, g.out_h))
            cc = 1 if cfg.grayscale else 3
            out = np.full(dw * dh * cc + 7, SENTINEL, np.uint8)
            orig = np.full(dw * dh * 3 + 7, SENTINEL, np.uint8)
            info = capi.McChainInfo()
            m = a.magnifier
            st = lib.mc_chain_process_yuv422(m._h, C.byref(capi.McYuv422(host.ctypes.data, pitch, 0, capi.MC_YUV422_YUYV)), w, h,
                                             C.byref(_to_mc(cfg)), int(cfg.grayscale), out.ctypes.data, out.size,
                                             orig.ctypes.data, orig.size, C.byref(info))
            assert st == capi.MC_OK
            fr = L.Frame(image=seen)
            cur, original = b.run_chain_once(fr, cfg)
            assert info_tuple(info)[:-1] == (0, dw, dh, cc, 0, dw, dh, 3)
            assert bool(info.magnified) == bool(b.magnifier.lane_produced()[0])
            assert np.array_equal(out[:-7], cur.image.reshape(-1)) and (out[-7:] == SENTINEL).all(), t
            assert np.array_equal(orig[:-7], original.image.reshape(-1)) and (orig[-7:] == SENTINEL).all(), t
            ccur, corig = c.run_chain_once(L.Frame(image=x.reshape(h, w, 2), format="YUYV", seq=t), cfg)
            assert ccur.seq == t and ccur.format == ("Gray8" if cc == 1 else "BGR8") and corig.format == "BGR8"
            assert np.array_equal(ccur.image, cur.image) and np.array_equal(corig.image, original.image), t
        for n_, l in state_names(b.magnifier, mode):
            assert np.array_equal(a.magnifier.get_state(n_, l), b.magnifier.get_state(n_, l)), (n_, l)
    finally:
        for p in keep:
            lib.mc_host_free(p)


# ---- errors ----------------------------------------------------------------------------------------------------------

def test_errors_return_before_any_launch_or_copy():
    """Every bad call is MC_ERR_INVALID (Color's refusal with a held lane MC_ERR_UNSUPPORTED) with the launch count, the
    outputs, the canvases and the state unchanged"""
    w, h, lanes = 130, 74, 2
    cfg = chain_cfg(O.MODE_LAPLACE, MODES["laplace"][1], down=2, gray=True)
    lay = Yuv(w, h, capi.MC_YUV422_YUYV)
    x = np.stack([from_bgr(lane_frame(0, k, w, h, 3), lay.order) for k in range(lanes)])
    d_in = Dev(lay.pack(x))
    lib, p = capi.lib(), _to_mc(cfg)
    ch = L.ProcessingChainB200(0, lanes=lanes)
    yuv_device_call(ch, cfg, x, 1, lay)   # state to keep
    m = ch.magnifier
    names = state_names(m, O.MODE_LAPLACE)
    before, n0 = [m.get_state(n, l) for n, l in names], m.launch_count
    out_step, orig_step = (w // 2), 3 * (w // 2)
    d_out, d_orig = Dev(np.full((2 * lanes, h // 2, out_step), SENTINEL, np.uint8)), Dev(np.full((2 * lanes, h // 2, orig_step), SENTINEL, np.uint8))
    cv = Canvas(capi.MC_CANVAS_BGR, *L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, capi.MC_SPLIT_LEFT_RIGHT), 2 * lanes)
    good = lay.struct(d_in.ptr)
    flags = np.zeros((2, lanes), np.uint8)
    base = dict(yv=good, frames=1, w=w, h=h, d_out=d_out.ptr, out_step=out_step, d_orig=d_orig.ptr, orig_step=orig_step,
                flags=flags, canvas=cv.struct(), split=capi.MC_SPLIT_LEFT_RIGHT)
    bad = [dict(yv=None), dict(yv=lay.struct(d_in.ptr, data=None)), dict(yv=lay.struct(d_in.ptr, order=2)),
           dict(yv=lay.struct(d_in.ptr, order=-1)), dict(w=w - 1), dict(w=0), dict(h=0),
           dict(yv=lay.struct(d_in.ptr, pitch=2 * w - 1)), dict(yv=lay.struct(d_in.ptr, lane_stride=2 * w * h - 1)),
           dict(frames=0), dict(frames=capi.MC_MAX_LANES), dict(flags=None), dict(out_step=out_step - 1),
           dict(orig_step=orig_step - 1), dict(d_out=None), dict(split=3), dict(canvas=cv.struct(data=None)),
           dict(canvas=cv.struct(pitch=3 * cv.cw - 1)), dict(canvas=cv.struct(lane_stride=1))]
    compose_only = ("split", "canvas")
    for bd in bad:
        args = {**base, **bd}
        info = capi.McChainInfo()
        yv = C.byref(args["yv"]) if args["yv"] is not None else None
        u8 = args["flags"].ctypes.data_as(C.POINTER(C.c_uint8)) if args["flags"] is not None else None
        if not any(k in bd for k in compose_only):
            assert lib.mc_chain_process_yuv422_device(m._h, yv, args["frames"], args["w"], args["h"], C.byref(p), 1,
                                                      args["d_out"], args["out_step"], args["d_orig"], args["orig_step"], u8,
                                                      C.byref(info)) == capi.MC_ERR_INVALID, bd
        if not any(k in bd for k in ("out_step", "orig_step", "d_out")):
            assert lib.mc_chain_compose_yuv422_device(m._h, yv, args["frames"], args["w"], args["h"], C.byref(p), 1,
                                                      args["split"], C.byref(args["canvas"]), u8,
                                                      C.byref(info)) == capi.MC_ERR_INVALID, bd
    m.sync()
    assert m.launch_count == n0
    assert (d_out.numpy() == SENTINEL).all() and (d_orig.numpy() == SENTINEL).all() and (cv.dev.numpy() == SENTINEL).all()
    assert all(np.array_equal(m.get_state(n, l), a) for (n, l), a in zip(names, before))

    # the host call: a 2-lane handle, and a bad argument on a 1-lane one, leave the outputs and the state alone
    one = L.ProcessingChainB200(0)
    host = np.ascontiguousarray(x[0])
    hy = capi.McYuv422(host.ctypes.data, 2 * w, 0, capi.MC_YUV422_YUYV)
    yuv_call = lambda hh, yv, ww, out_n, orig_n, prm=p: lib.mc_chain_process_yuv422(
        hh, C.byref(yv) if yv is not None else None, ww, h, C.byref(prm), 1, o.ctypes.data, out_n, g.ctypes.data, orig_n,
        C.byref(capi.McChainInfo()))
    o, g = np.full(h * w, SENTINEL, np.uint8), np.full(h * w * 3, SENTINEL, np.uint8)
    fo, fg = (w // 2) * (h // 2), 3 * (w // 2) * (h // 2)
    assert yuv_call(m._h, hy, w, fo, fg) == capi.MC_ERR_INVALID
    one_n0 = one.magnifier.launch_count
    bad_mode = _to_mc(cfg)
    bad_mode.mode = 7
    for args in [(None, w, fo, fg), (capi.McYuv422(None, 2 * w, 0, 0), w, fo, fg), (capi.McYuv422(host.ctypes.data, 2 * w, 0, 5), w, fo, fg),
                 (hy, w - 1, fo, fg), (capi.McYuv422(host.ctypes.data, 2 * w - 2, 0, 0), w, fo, fg), (hy, w, fo - 1, fg),
                 (hy, w, fo, fg - 1)]:
        assert yuv_call(one.magnifier._h, *args) == capi.MC_ERR_INVALID, args
    assert yuv_call(one.magnifier._h, hy, w, fo, fg, bad_mode) == capi.MC_ERR_INVALID
    assert one.magnifier.launch_count == one_n0 and (o == SENTINEL).all() and (g == SENTINEL).all()

    # Color refuses a held lane across a multi-lane handle, as the BGR call does
    color = chain_cfg(O.MODE_COLOR, MODES["color"][1], down=2, gray=True)
    cch = L.ProcessingChainB200(0, lanes=lanes)
    yuv_device_call(cch, color, x, 1, lay)
    cch.magnifier.hold_lane(1, True)
    n1 = cch.magnifier.launch_count
    info = capi.McChainInfo()
    assert lib.mc_chain_process_yuv422_device(cch.magnifier._h, C.byref(good), 1, w, h, C.byref(_to_mc(color)), 1, d_out.ptr,
                                              out_step, d_orig.ptr, orig_step, flags.ctypes.data_as(C.POINTER(C.c_uint8)),
                                              C.byref(info)) == capi.MC_ERR_UNSUPPORTED
    cch.magnifier.sync()
    assert cch.magnifier.launch_count == n1 and (d_out.numpy() == SENTINEL).all()
