"""RGB frames into the chain and RGB export canvases: mc_chain_process_rgb_device, mc_chain_compose_rgb_device,
mc_chain_submit_rgb, mc_chain_compose_submit_rgb, MC_CANVAS_RGB and MC_CANVAS_RGB_PLANAR.

For any RGB-family input X (packed RGB, RGBA, BGRA or three planes) a call must equal, bit for bit, the BGR call on
B = cv2.cvtColor(X, COLOR_RGB2BGR / RGBA2BGR / BGRA2BGR) (planar: cv2.merge of the B, G, R planes): flags, lane flags,
processed frames, original tap and temporal state.  The conversion is a front stage that always runs, as for 4:2:2, so
test_gpu_yuv422's checkers take RGB frames in place of 4:2:2 ones, against a twin handle's BGR calls.  An RGB canvas
must be the BGR canvas of the same call with its channels swapped (planar: as three planes); buffers are sentinel-filled,
so bytes written where they should not be (row padding, the 4th byte of a pixel, space after the planes) show up."""
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
import test_gpu_chain_submit as chain_submit
import test_gpu_compose_submit as compose_submit
import test_gpu_yuv422 as yuv422
import test_gpu_yuv420p as yuv420p
from test_gpu_chain_lanes import MODES, chain_cfg, device_call, info_tuple, none_cfg
from test_gpu_compose import SPLITS, Canvas
from test_gpu_lanes import SENTINEL, lane_frame
from test_gpu_nv12 import Dev, Layout, to_nv12
from test_gpu_yuv422 import Yuv, from_bgr as yuyv_of, yuv_device_call   # bound here: rgb_frames patches the module

pytestmark = pytest.mark.gpu

EMU = os.environ.get("MC_EMU") == "1"
RGB, RGBA, BGRA, PLANAR = capi.MC_RGB_RGB, capi.MC_RGB_RGBA, capi.MC_RGB_BGRA, capi.MC_RGB_PLANAR
LAYOUTS = {"rgb": RGB, "rgba": RGBA, "bgra": BGRA, "planar": PLANAR}
BPP = {RGB: 3, RGBA: 4, BGRA: 4, PLANAR: 1}
BGR_C, NV12_C, I420_C = capi.MC_CANVAS_BGR, capi.MC_CANVAS_NV12, capi.MC_CANVAS_I420
RGB_C, PLANAR_C = capi.MC_CANVAS_RGB, capi.MC_CANVAS_RGB_PLANAR
NONE, LR, TB = capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM


# ---- RGB frames, as PyTorch, image libraries and desktop capture hand them out ----------------------------------------

def from_bgr(bgr, layout):
    """BGR [h][w][3] -> the frame of that layout: packed [h][w * bpp] (the 4th byte a pattern nothing may read) or
    planar [3][h][w] (R, G, B)"""
    h, w = bgr.shape[:2]
    if layout == PLANAR:
        return np.stack([bgr[..., 2], bgr[..., 1], bgr[..., 0]])
    px = bgr if layout == BGRA else bgr[..., ::-1]
    if layout != RGB:
        alpha = ((np.arange(h * w, dtype=np.uint32) * 97 + 13) & 255).astype(np.uint8).reshape(h, w, 1)
        px = np.concatenate([px, alpha], -1)
    return np.ascontiguousarray(px).reshape(h, -1)


CODES = {RGB: cv2.COLOR_RGB2BGR, RGBA: cv2.COLOR_RGBA2BGR, BGRA: cv2.COLOR_BGRA2BGR}


def convert(x, layout):
    """cv2's BGR of frames x [V](frame) of that layout -> [V][h][w][3]"""
    out = []
    for f in x:
        if layout == PLANAR:
            out.append(cv2.merge([np.ascontiguousarray(f[2]), np.ascontiguousarray(f[1]), np.ascontiguousarray(f[0])]))
        else:
            h = f.shape[0]
            out.append(cv2.cvtColor(np.ascontiguousarray(f).reshape(h, -1, BPP[layout]), CODES[layout]))
    return np.stack(out)


class Rgb:
    """Where an RGB frame set sits: lanes blocks, `offset` bytes from the buffer's start; rows `pitch` bytes apart (packed
    >= w * bpp, planar >= w) and `lane_rows` spare rows after each frame.  Planar arrangements: "rgb" (the planes one
    after the other), "bgr" (in reversed memory order) or "far" (a long way apart, `gap` bytes between)."""

    def __init__(self, w, h, layout, pitch=None, lane_rows=0, offset=0, arrangement="rgb", gap=0):
        self.w, self.h, self.layout = w, h, layout
        self.pitch = pitch or w * BPP[layout]
        assert self.pitch >= w * BPP[layout]
        plane = self.pitch * (h + lane_rows)
        if layout != PLANAR:
            self.ofs, self.block = (0,), plane
        elif arrangement == "rgb":
            self.ofs, self.block = (0, plane + gap, 2 * plane + 2 * gap), 3 * plane + 3 * gap
        elif arrangement == "bgr":
            self.ofs, self.block = (2 * plane + 2 * gap, plane + gap, 0), 3 * plane + 3 * gap
        else:
            self.ofs = (0, plane + 8192 + gap, 2 * plane + 3 * gap + 20000)
            self.block = self.ofs[2] + plane + gap
        self.offset = offset

    @property
    def lane_stride(self):
        return self.block

    def pack(self, x, fill=0x3C):
        buf = np.full(len(x) * self.block + self.offset, fill, np.uint8)
        row = self.w * BPP[self.layout]
        for v, f in enumerate(x):
            planes = f if self.layout == PLANAR else f[None]
            for o, p in zip(self.ofs, planes):
                base = self.offset + v * self.block + o
                buf[base:base + self.h * self.pitch].reshape(self.h, self.pitch)[:, :row] = p
        return buf

    def struct(self, base, **override):
        ptrs = [base + self.offset + o for o in self.ofs]
        f = dict(data=ptrs[0], g=ptrs[1] if self.layout == PLANAR else None, b=ptrs[2] if self.layout == PLANAR else None,
                 pitch=self.pitch, lane_stride=self.block, layout=self.layout)
        f.update(override)
        return capi.McRgb(f["data"], f["g"], f["b"], f["pitch"], f["lane_stride"], f["layout"])


def rgb_device_call(ch, cfg, x, frames, lay, out_pad=0, orig_pad=0, want_orig=True):
    """one mc_chain_process_rgb_device call on frames x -> (flags, info, out, orig), test_gpu_yuv422.yuv_device_call's
    buffers"""
    g = ch.geometry(cfg, lay.w, lay.h, 3)
    dw, dh = (lay.w, lay.h) if g.cur_is_input and g.orig_is_input else (
        (g.orig_w, g.orig_h) if not g.orig_is_input else (g.out_w, g.out_h))
    cc = 1 if cfg.grayscale else 3
    v = len(x)
    out_step, orig_step = dw * cc + out_pad, dw * 3 + orig_pad
    d_in = Dev(lay.pack(x))
    d_out = Dev(np.full((v, dh, out_step), SENTINEL, np.uint8))
    d_orig = Dev(np.full((v, dh, orig_step), SENTINEL, np.uint8)) if want_orig else None
    flags, info = ch.process_rgb_device(lay.struct(d_in.ptr), frames, lay.w, lay.h, cfg, d_out.ptr, out_step,
                                        d_orig.ptr if d_orig else 0, orig_step)
    ch.magnifier.sync()
    return flags.astype(np.uint8), info, d_out.numpy(), d_orig.numpy() if d_orig else None


@pytest.fixture()
def rgb_frames(monkeypatch):
    """test_gpu_yuv422's chain checker with RGB frames: its `order` is the mc_rgb_layout, its layout class Rgb"""
    monkeypatch.setattr(yuv422, "from_bgr", from_bgr)
    monkeypatch.setattr(yuv422, "convert", convert)
    monkeypatch.setattr(yuv422, "Yuv", Rgb)
    monkeypatch.setattr(yuv422, "yuv_device_call", rgb_device_call)


# ---- the front ----------------------------------------------------------------------------------------------------------

def every_colour(w, h):
    """-> BGR [h][w][3] whose first 2^24 pixels (w * h >= 2^24) hold every (B, G, R) triple once"""
    i = np.arange(w * h, dtype=np.uint32) % (1 << 24)
    return np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(h, w, 3)


@pytest.mark.skipif(EMU, reason="every colour is too slow for the CPU emulation")
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("w,h,lay_kw", [
    (4096, 4096, dict()),                                                         # tight rows, 8-byte aligned
    (4096, 4096, dict(pitch_pad=64, arrangement="bgr", lane_rows=1)),            # padded, planes in reversed order
    (4090, 4093, dict(pitch_pad=3, offset=1, arrangement="far", gap=5)),          # odd pitch and base, planes far apart
], ids=["tight", "padded_reversed", "odd_far"])
def test_front_and_compose_on_every_colour(layout, w, h, lay_kw):
    """Mode None with a full-frame ROI and grayscale: d_original is cv2's conversion and d_out its gray (the front), and
    an MC_SPLIT_NONE BGR canvas is the conversion cropped to even size (the compose)"""
    o = LAYOUTS[layout]
    kw = dict(lay_kw)
    pad = kw.pop("pitch_pad", 0)
    lay = Rgb(w, h, o, pitch=w * BPP[o] + pad, **kw)
    want = every_colour(w, h)
    x = from_bgr(want, o)[None]
    assert np.array_equal(convert(x, o)[0], want)
    ch = L.ProcessingChainB200(0)
    flags, info, out, orig = rgb_device_call(ch, none_cfg(roi=(0.0, 0.0, 1.0, 1.0), gray=True), x, 1, lay, 2, 6)
    assert not flags.any() and info_tuple(info) == (0, w, h, 1, 0, w, h, 3, 0)
    assert np.array_equal(orig[0][:, :3 * w], want.reshape(h, 3 * w)) and (orig[0][:, 3 * w:] == SENTINEL).all()
    assert np.array_equal(out[0][:, :w], cv2.cvtColor(want, cv2.COLOR_BGR2GRAY)) and (out[0][:, w:] == SENTINEL).all()
    for fmt in (BGR_C, RGB_C, PLANAR_C):
        cv = CanvasRgb(fmt, w & ~1, h & ~1, 1, pad=8)
        d_in = Dev(lay.pack(x))
        ch.magnifier.chain_compose_rgb_device(lay.struct(d_in.ptr), 1, w, h, none_cfg(), NONE, cv.struct())
        ch.magnifier.sync()
        assert np.array_equal(cv.dev.numpy(), cv.expected([want[:h & ~1, :w & ~1]])), fmt


W, H = (46, 31) if EMU else (134, 77)   # odd height
FRONT_CASES = [dict(), dict(gray=True), dict(roi=(0.015, 0.013, 0.5, 0.8)), dict(down=2), dict(down=3), dict(down=8),
               dict(down=3, roi=(0.1, 0.15, 0.8, 0.75), gray=True)]   # ROI at an odd column and row; fractional area


@pytest.mark.parametrize("settings", FRONT_CASES, ids=["none", "gray", "roi_odd", "down2", "down3", "down8", "roi_down3_gray"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_front_matches_the_bgr_front(rgb_frames, layout, settings):
    """Mode None over 3 lanes x 2 frames, rows padded to an odd pitch from an odd base"""
    o = LAYOUTS[layout]
    yuv422.check_yuv(O.MODE_NONE, MODES["laplace"][1], W, H, [("cfg", settings), ("clip", 2), ("frame",)], lanes=3, order=o,
                     lay_kw=dict(pitch=W * BPP[o] + 5, lane_rows=1, offset=1, arrangement="far", gap=3), pads=(3, 5))


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("settings", [dict(), dict(gray=True), dict(down=2), dict(roi=(0.015, 0.013, 0.6, 0.8))],
                         ids=["none", "gray", "down2", "roi_odd"])
@pytest.mark.parametrize("lanes", [1, 3])
def test_chain_equals_bgr_chain_on_cv2_conversion(rgb_frames, mname, settings, lanes):
    """frames and clips of 1, 3 and 16; restart and hold on 3 lanes (not Color, which refuses them across lanes);
    planar frames on 3 lanes, RGBA on 1"""
    mode, ui = MODES[mname]
    lifecycle = [] if mname == "color" or lanes == 1 else [("restart", 2), ("hold", 1, 1), ("frame",), ("clip", 3), ("hold", 1, 0)]
    steps = [("cfg", settings), ("frame",), ("clip", 3), *lifecycle, ("clip", 16 if not EMU else 2), ("frame",), ("clip", 1)]
    o = PLANAR if lanes == 3 else RGBA
    yuv422.check_yuv(mode, ui, W, H, steps, lanes=lanes, order=o, lay_kw=dict(pitch=W * BPP[o] + 64))


@pytest.mark.parametrize("mname", list(MODES))
def test_lane_params_and_color_lifecycle(mname):
    """restart, hold and per-lane parameters on 3 lanes (Color with color_lane_lifecycle): the RGB handle against the
    I420 checker's twins fed cv2's conversion (frames, taps, info, flags and state)"""
    mode, ui = MODES[mname]
    check_rgb_twins(mode, ui, [("frame",), ("restart", 2), ("hold", 1, 1), ("clip", 3), ("hold", 1, 0), ("lp", 0),
                               ("clip", 16 if not EMU else 2), ("frame",)], lanes=3, layout=BGRA)


@pytest.mark.parametrize("mname", list(MODES))
def test_rgb_bgr_nv12_yuyv_and_i420_calls_interleave(mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("nv12",), ("frame",), ("yuyv",), ("clip", 3), ("bgr",), ("i420",), ("frame",), ("cfg", dict(down=2)),
             ("frame",), ("nv12",), ("i420",), ("frame",)]
    check_rgb_twins(mode, ui, steps, lanes=2, layout=RGB, h=H + H % 2)   # NV12 and I420 need an even height


def check_rgb_twins(mode, ui, steps, lanes, layout, w=W, h=H):
    """Handle A takes RGB calls, B the BGR calls on cv2's conversion; ("nv12",) / ("yuyv",) / ("bgr",) / ("i420",) steps
    run that call on both, which must agree.  ("restart", k) / ("hold", k, on) / ("lp", k) on both."""
    cfg = chain_cfg(mode, ui)
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    if mode == O.MODE_COLOR:
        for ch in (a, b):
            ch.magnifier.set_option("color_lane_lifecycle", 1)
    lay = Rgb(w, h, layout, pitch=w * BPP[layout] + 2)
    held, t = [False] * lanes, 0
    for step in steps:
        if step[0] in ("restart", "hold", "lp"):
            for ch in (a, b):
                if step[0] == "restart":
                    ch.magnifier.restart_lane(step[1])
                elif step[0] == "hold":
                    ch.magnifier.hold_lane(step[1], step[2])
                else:
                    ch.set_lane_params(step[1], dataclasses.replace(cfg.magnification, amplification=cfg.magnification.amplification + 7))
            if step[0] == "hold":
                held[step[1]] = bool(step[2])
            continue
        if step[0] == "cfg":
            cfg = chain_cfg(mode, ui, **step[1])
            continue
        n = step[1] if step[0] == "clip" else 1
        bgr = np.stack([lane_frame(s, k, w, h, 3) for s in range(t, t + n) for k in range(lanes)])
        t += n
        if step[0] in ("nv12", "yuyv", "bgr", "i420"):
            rs = []
            for ch in (a, b):
                if step[0] == "nv12":
                    rs.append(device_call(ch, cfg, np.stack([to_nv12(f) for f in bgr]), n, w, h, 3, nv12=Layout(w, h)))
                elif step[0] == "bgr":
                    rs.append(device_call(ch, cfg, bgr, n, w, h, 3))
                elif step[0] == "i420":
                    rs.append(yuv420p.i420_call(ch, cfg, np.stack([yuv420p.to_i420(f) for f in bgr]), n, yuv420p.Lay(w, h)))
                else:
                    yl = Yuv(w, h, capi.MC_YUV422_YUYV)
                    rs.append(yuv_device_call(ch, cfg, np.stack([yuyv_of(f, capi.MC_YUV422_YUYV) for f in bgr]), n, yl))
            assert np.array_equal(rs[0][0], rs[1][0]) and info_tuple(rs[0][1]) == info_tuple(rs[1][1]), step
            assert np.array_equal(rs[0][2], rs[1][2]) and np.array_equal(rs[0][3], rs[1][3]), step
            continue
        x = np.stack([from_bgr(f, layout) for f in bgr])
        seen = convert(x, layout)
        flags, info, out, orig = rgb_device_call(a, cfg, x, n, lay, 3, 5)
        bflags, binfo, bout, borig = device_call(b, cfg, seen, n, w, h, 3)
        assert np.array_equal(flags, bflags), step
        assert info_tuple(info) == yuv422.yuv_info(binfo, w, h, cfg.grayscale), step
        assert np.array_equal(a.magnifier.lane_produced(), b.magnifier.lane_produced()), step
        (orows, _), (grows, _) = yuv422.out_geom(b, cfg, w, h, 3)
        outs, origs = [], []
        for v in range(n * lanes):
            if held[v % lanes]:
                outs.append(None)
                origs.append(None)
                continue
            outs.append(seen[v] if binfo.cur_is_input and not bflags.ravel()[v] else
                        yuv422.image(bout[v], orows, info.out_w, info.out_channels))
            origs.append(seen[v] if binfo.orig_is_input else yuv422.image(borig[v], grows, info.orig_w, 3))
        assert np.array_equal(out, yuv422.filled(out, info.out_w * info.out_channels, outs)), step
        assert np.array_equal(orig, yuv422.filled(orig, info.orig_w * 3, origs)), step
    yuv420p.assert_same_state(a, b, mode)
    return a


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
@pytest.mark.parametrize("mname", list(MODES))
def test_1080p(rgb_frames, mname):
    mode, ui = MODES[mname]
    yuv422.check_yuv(mode, ui, 1920, 1080, [("frame",), ("frame",), ("clip", 3), ("frame",)], order=PLANAR)


# ---- canvases ---------------------------------------------------------------------------------------------------------

class CanvasRgb(Canvas):
    """Canvas with the RGB formats as well: packed RGB rows of 3 * cw + pad bytes, or the R, G and B planes of ch rows of
    cw + pad bytes one after the other; `lane_rows` spare rows after each lane."""

    def __init__(self, fmt, cw, ch, v, pad=0, lane_rows=0, uv_gap=0):
        if fmt not in (RGB_C, PLANAR_C):
            return super().__init__(fmt, cw, ch, v, pad, lane_rows, uv_gap) if fmt != I420_C else \
                yuv420p.Canvas420.__init__(self, fmt, cw, ch, v, pad, lane_rows, uv_gap)
        self.fmt, self.cw, self.ch, self.uv_row = fmt, cw, ch, None
        self.pitch = (3 * cw if fmt == RGB_C else cw) + pad
        self.rows = (ch if fmt == RGB_C else 3 * ch) + lane_rows
        self.dev = Dev(np.full((v, max(self.rows, 1), max(self.pitch, 1)), SENTINEL, np.uint8))

    def expected(self, canvases):
        if self.fmt == I420_C:
            return yuv420p.Canvas420.expected(self, canvases)
        if self.fmt not in (RGB_C, PLANAR_C):
            return super().expected(canvases)
        want = np.full((len(canvases), max(self.rows, 1), max(self.pitch, 1)), SENTINEL, np.uint8)
        for v, im in enumerate(canvases):
            if im is not None:
                put_rgb(want[v], self, im)
        return want


def put_rgb(lane, cv, bgr):
    """a BGR canvas image as canvas cv's format into one lane [rows][pitch]"""
    if cv.fmt == RGB_C:
        lane[:cv.ch, :3 * cv.cw] = bgr[..., ::-1].reshape(cv.ch, 3 * cv.cw)
    else:
        for k in range(3):
            lane[k * cv.ch:(k + 1) * cv.ch, :cv.cw] = bgr[..., 2 - k]


def swap_canvas(bgr_lanes, bgr_cv, cv, written):
    """the canvas cv (RGB format) holding BGR canvas bgr_cv's lanes with their channels swapped, for the lanes written"""
    want = np.full((len(written), max(cv.rows, 1), max(cv.pitch, 1)), SENTINEL, np.uint8)
    for v, wr in enumerate(written):
        if wr and cv.cw:
            put_rgb(want[v], cv, bgr_lanes[v, :cv.ch, :3 * cv.cw].reshape(cv.ch, cv.cw, 3))
    return want


def compose_rgb(m, cfg, xs, n, lay, split, cv):
    d_in = Dev(lay.pack(xs))
    flags, info = m.chain_compose_rgb_device(lay.struct(d_in.ptr), n, lay.w, lay.h, cfg, split, cv.struct())
    m.sync()
    return flags.astype(np.uint8), info


def check_compose_rgb(mode, ui, w, h, fmt, split, steps, lanes=1, src="rgb", layout=RGB, labels=False, lay_kw=None, pad=6,
                      lane_rows=1):
    """Handle A composes `src` frames into `fmt` canvases; its twin B composes the same content, as BGR frames into BGR
    canvases for an RGB source, or as the same source into a BGR canvas for the others.  A's canvas must be B's, with
    its channels swapped for an RGB format; A's flags, info and lane flags B's, with info as for 4:2:2 (both frames
    written) for an RGB source."""
    cfg = chain_cfg(mode, ui)
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    lay = Rgb(w, h, layout, **(lay_kw or {}))
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
        v = n * lanes
        c = 1 if src == "gray" else 3
        cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, c, split)
        if labels and cw:
            for ch in (a, b):
                ch.magnifier.set_overlay(export_labels(cw, chh, split))
        rgb_fmt = fmt in (RGB_C, PLANAR_C)
        cva = CanvasRgb(fmt, cw, chh, v, pad, lane_rows, 3)
        cvb = CanvasRgb(BGR_C if rgb_fmt else fmt, cw, chh, v, pad, lane_rows, 3)
        if src == "rgb":
            xs = np.stack([from_bgr(f, layout) for f in bgr])
            ra = compose_rgb(a.magnifier, cfg, xs, n, lay, split, cva)
            d_b = Dev(convert(xs, layout))
            rb = b.magnifier.chain_compose_device(d_b.ptr, n, w, h, 3, 3 * w, cfg, split, cvb.struct())
        else:
            if src == "nv12":
                nv = Layout(w, h, pitch=w + 4, uv_row=h + 2)
                d = Dev(nv.pack(np.stack([to_nv12(f) for f in bgr]), fill=0x3C))
                call = lambda m, cv: m.chain_compose_nv12_device(nv.planes(d.ptr), n, w, h, cfg, split, cv.struct())
            elif src == "i420":
                il = yuv420p.Lay(w, h, pitch=w + 2)
                d = Dev(il.pack(np.stack([yuv420p.to_i420(f) for f in bgr])))
                call = lambda m, cv: m.chain_compose_yuv420p_device(il.struct(d.ptr), n, w, h, cfg, split, cv.struct())
            elif src == "yuyv":
                yl = Yuv(w, h, capi.MC_YUV422_YUYV, pitch=2 * w + 2)
                d = Dev(yl.pack(np.stack([yuyv_of(f, capi.MC_YUV422_YUYV) for f in bgr])))
                call = lambda m, cv: m.chain_compose_yuv422_device(yl.struct(d.ptr), n, w, h, cfg, split, cv.struct())
            else:
                frames = bgr if c == 3 else np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr])
                d = Dev(frames)
                call = lambda m, cv: m.chain_compose_device(d.ptr, n, w, h, c, w * c, cfg, split, cv.struct())
            ra, rb = call(a.magnifier, cva), call(b.magnifier, cvb)
        a.magnifier.sync()
        b.magnifier.sync()
        assert np.array_equal(np.asarray(ra[0]).astype(np.uint8), np.asarray(rb[0]).astype(np.uint8)), step
        binfo = info_tuple(rb[1])
        if src == "rgb":
            binfo = yuv422.yuv_info(rb[1], w, h, cfg.grayscale)
        assert info_tuple(ra[1]) == binfo, (step, info_tuple(ra[1]), binfo)
        assert np.array_equal(a.magnifier.lane_produced(), b.magnifier.lane_produced()), step
        got, ref = cva.dev.numpy(), cvb.dev.numpy()
        if rgb_fmt:
            ref = swap_canvas(ref, cvb, cva, [not held[k % lanes] and cw > 0 for k in range(v)])
        assert np.array_equal(got, ref), (step, np.argwhere(got != ref)[:5])
    yuv420p.assert_same_state(a, b, mode)


@pytest.mark.parametrize("fmt", [BGR_C, NV12_C, I420_C, RGB_C, PLANAR_C], ids=["bgr", "nv12", "i420", "rgb", "planar"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_rgb_sources_into_every_canvas(layout, fmt):
    """labels, a held lane, a ROI, a downscale and grayscale; frames at an odd base and pitch; the split cycles over the
    cases"""
    split = list(SPLITS)[(list(LAYOUTS).index(layout) + fmt) % 3]
    steps = [("frame",), ("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 3), ("hold", 1, 1), ("cfg", dict(down=2)),
             ("frame",), ("hold", 1, 0), ("restart", 0), ("cfg", dict(gray=True)), ("clip", 2)]
    o = LAYOUTS[layout]
    check_compose_rgb(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, SPLITS[split], steps, lanes=2, layout=o,
                      labels=split != "none", lay_kw=dict(pitch=W * BPP[o] + 3, offset=1, arrangement="bgr"))


@pytest.mark.parametrize("fmt", [RGB_C, PLANAR_C], ids=["rgb_canvas", "planar_canvas"])
@pytest.mark.parametrize("src", ["bgr", "gray", "nv12", "yuyv", "i420", "rgb"])
@pytest.mark.parametrize("split", list(SPLITS))
def test_rgb_canvases_from_every_source(split, src, fmt):
    """labels included; row padding and the rows after the planes stay sentinel"""
    steps = [("frame",), ("clip", 3), ("cfg", dict(down=2)), ("frame",)]
    check_compose_rgb(O.MODE_LAPLACE, MODES["laplace"][1], W, H + H % 2, fmt, SPLITS[split], steps, src=src, labels=True,
                      pad=10, lane_rows=2)


@pytest.mark.parametrize("mname", ["phase", "color"])
@pytest.mark.parametrize("aligned", [True, False], ids=["vec", "bytes"])
@pytest.mark.parametrize("fmt", [RGB_C, PLANAR_C], ids=["rgb_canvas", "planar_canvas"])
def test_rgb_canvas_frames_not_produced(fmt, mname, aligned):
    """Phase's first frame and Color's warm-up compose the front's output; 8-byte aligned canvases or the byte path"""
    mode, ui = MODES[mname]
    check_compose_rgb(mode, ui, 64, 32, fmt, LR, [("frame",), ("clip", 3), ("frame",)], layout=PLANAR,
                      pad=0 if aligned else 5, lane_rows=0 if aligned else 1,
                      lay_kw=None if aligned else dict(pitch=66, offset=1))


@pytest.mark.parametrize("fmt", [RGB_C, PLANAR_C], ids=["rgb_canvas", "planar_canvas"])
def test_empty_rgb_canvas_writes_nothing(fmt):
    """a 1 x 1 chain output has a 0 x 0 canvas: nothing is written"""
    cfg = chain_cfg(O.MODE_LAPLACE, MODES["laplace"][1], down=8)
    w, h = 14, 12
    assert L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR) == (0, 0)
    ch = L.ProcessingChainB200(0)
    buf = Dev(np.full((1, 4, 8), SENTINEL, np.uint8))
    lay = Rgb(w, h, RGB)
    d_in = Dev(lay.pack(from_bgr(lane_frame(0, 0, w, h, 3), RGB)[None]))
    ch.magnifier.chain_compose_rgb_device(lay.struct(d_in.ptr), 1, w, h, cfg, LR, capi.McCanvas(fmt, buf.ptr, None, 2, 32))
    ch.magnifier.sync()
    assert (buf.numpy() == SENTINEL).all()


# ---- submits: the pipelined checkers of the other sources, with RGB frames and canvases ------------------------------

SUB_LAYOUT = {"rgb": RGB, "rgba": RGBA, "bgra": BGRA, "planar": PLANAR}


class ChainSource(yuv420p.ChainSource):
    def __init__(self, kind, lanes, w, h, pad):
        if kind not in SUB_LAYOUT:
            return super().__init__(kind, lanes, w, h, pad)
        self.kind, self.lanes, self.w, self.h, self.c = kind, lanes, w, h, 3
        o = SUB_LAYOUT[kind]
        self.lay = Rgb(w, h, o, pitch=w * BPP[o] + pad, lane_rows=1 if pad else 0, arrangement="bgr" if pad else "rgb")

    def frame(self, t):
        if self.kind not in SUB_LAYOUT:
            return super().frame(t)
        return self.lay.pack(np.stack([from_bgr(lane_frame(t, k, self.w, self.h, 3), self.lay.layout) for k in range(self.lanes)]))

    def device_call(self, ch, cfg, d_in, d_out, out_step, d_orig, orig_step):
        if self.kind not in SUB_LAYOUT:
            return super().device_call(ch, cfg, d_in, d_out, out_step, d_orig, orig_step)
        return ch.process_rgb_device(self.lay.struct(d_in), 1, self.w, self.h, cfg, d_out, out_step, d_orig, orig_step)

    def submit(self, ch, cfg, base, out, out_step, orig, orig_step):
        if self.kind not in SUB_LAYOUT:
            return super().submit(ch, cfg, base, out, out_step, orig, orig_step)
        return ch.submit_rgb(self.lay.struct(base), self.w, self.h, cfg, out, out_step, orig, orig_step)

    def geometry(self, cfg):
        out, orig, front = super().geometry(cfg)
        if self.kind not in SUB_LAYOUT:
            return out, orig, front
        g = L.ProcessingChainB200.geometry(cfg, self.w, self.h, 3)   # the conversion always runs, as for 4:2:2
        dw, dh = (self.w, self.h) if g.cur_is_input and g.orig_is_input else (
            (g.orig_w, g.orig_h) if not g.orig_is_input else (g.out_w, g.out_h))
        return (dh, dw * (1 if cfg.grayscale else 3)), (dh, dw * 3), True


class ClipSource(yuv420p.ClipSource):
    def __init__(self, kind, lanes, w, h, pad):
        super().__init__("bgr" if kind in SUB_LAYOUT else kind, lanes, w, h, pad)
        if kind in SUB_LAYOUT:
            self.kind = kind
            o = SUB_LAYOUT[kind]
            self.lay = Rgb(w, h, o, pitch=w * BPP[o] + pad, arrangement="far" if pad else "rgb", gap=pad)

    def pack(self, bgr):
        if self.kind not in SUB_LAYOUT:
            return super().pack(bgr)
        return self.lay.pack(np.stack([from_bgr(f, self.lay.layout) for f in bgr]))

    def device_call(self, m, cfg, d_in, n, split, canvas):
        if self.kind not in SUB_LAYOUT:
            return super().device_call(m, cfg, d_in, n, split, canvas)
        return m.chain_compose_rgb_device(self.lay.struct(d_in), n, self.w, self.h, cfg, split, canvas)

    def submit(self, ch, cfg, base, n, split, canvas):
        if self.kind not in SUB_LAYOUT:
            return super().submit(ch, cfg, base, n, split, canvas)
        return ch.compose_submit_rgb(self.lay.struct(base), n, self.w, self.h, cfg, split, canvas)


@pytest.fixture()
def rgb_submits(monkeypatch):
    """the submit checkers of test_gpu_chain_submit / test_gpu_compose_submit, with RGB sources and canvases"""
    monkeypatch.setattr(chain_submit, "Source", ChainSource)
    monkeypatch.setattr(compose_submit, "ClipSource", ClipSource)
    monkeypatch.setattr(compose_submit, "Canvas", CanvasRgb)


@pytest.mark.parametrize("kind,front,depth", [("rgb", "none", 1), ("rgba", "roi", 3), ("bgra", "down2", 5), ("planar", "gray", 1),
                                              ("planar", "roi_down_gray", 3), ("rgb", "roi_down_gray", 5)])
def test_chain_submit_equals_the_device_chain(rgb_submits, kind, front, depth):
    """restarts, holds, an amplification change, a ROI move and a levels change in flight; pinned and pageable buffers"""
    pins = [(True, False, True), (False, True, False), (True, True, True)][depth // 2]
    chain_submit.check_chain_submit(kind, front, "laplace", lanes=3, depth=depth, pins=pins, n=14 if EMU else 20)


@pytest.mark.parametrize("kind,fmt,split,depth", [("rgb", RGB_C, LR, 1), ("planar", PLANAR_C, TB, 3), ("bgra", NV12_C, NONE, 5),
                                                  ("rgba", I420_C, LR, 1), ("planar", BGR_C, LR, 3), ("bgr", PLANAR_C, TB, 5),
                                                  ("nv12", RGB_C, NONE, 1), ("yuyv", PLANAR_C, LR, 3), ("i420", RGB_C, TB, 5),
                                                  ("gray", PLANAR_C, LR, 1), ("rgb", PLANAR_C, LR, 5)])
def test_compose_submit_equals_the_device_compose(rgb_submits, kind, fmt, split, depth):
    """clips of 16, 3 and 1 and a shorter last clip; an overlay set / replaced / cleared, restarts, holds, lane params, a ROI
    move and a levels change in flight; input and canvas pinned and pageable in turn"""
    clips = (4, 3, 1, 4, 2) if EMU else compose_submit.CLIPS
    compose_submit.check_compose_submit(kind, "roi" if depth != 3 else "down2", "laplace", lanes=2, depth=depth, clips=clips,
                                        fmt=fmt, split=split, pad=6)


@pytest.mark.parametrize("mname", ["phase", "color"])
def test_compose_submit_modes(rgb_submits, mname):
    compose_submit.check_compose_submit("planar", "gray", mname, lanes=3, depth=3, clips=(3, 2, 1, 3), fmt=PLANAR_C, split=LR)


def test_submits_interleave_in_fifo_order_with_nv12_and_yuyv(rgb_submits):
    """mc_chain_compose_submit_rgb, mc_chain_submit_rgb, mc_submit_nv12 and mc_chain_submit_yuv422 in turn on one handle,
    each collect equal to its own device call on a twin that runs them in the same order"""
    w, h, lanes = W, H + H % 2, 2
    cfg = chain_cfg(*MODES["laplace"])
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    srcs = {"yuyv": ChainSource("yuyv", lanes, w, h, 4), "rgb": ChainSource("bgra", lanes, w, h, 2)}
    cs = ClipSource("planar", lanes, w, h, 2)
    nvl = Layout(w, h, pitch=w + 2, uv_row=h + 1)
    lib, keep, pending, t = capi.lib(), [], [], 0
    try:
        for i in range(12):
            which = ("compose", "nv12", "yuyv", "rgb")[i % 4]
            if which == "nv12":
                x = np.stack([chain_submit.to_nv12(lane_frame(t, k, w, h, 3)) for k in range(lanes)])
                t += 1
                d_in, d_out = Dev(nvl.pack(x)), Dev(nvl.pack(np.zeros_like(x), fill=SENTINEL))
                st = lib.mc_process_nv12_device(twin.magnifier._h, C.byref(nvl.planes(d_in.ptr)), w, h, C.byref(_to_mc(cfg)),
                                                C.byref(nvl.planes(d_out.ptr)), C.byref(C.c_int()))
                assert st == capi.MC_OK
                host_in = chain_submit.host_buffer(d_in.numpy().shape, i % 2 == 0, lib, keep, 0)
                host_in[...] = nvl.pack(x)
                out = chain_submit.host_buffer(host_in.shape, False, lib, keep, SENTINEL)
                sub.magnifier.submit_nv12(nvl.planes(host_in.ctypes.data), w, h, cfg, nvl.planes(out.ctypes.data))
                outs, want = (out,), (d_out,)
            elif which in ("yuyv", "rgb"):
                src = srcs[which]
                frame = src.frame(t)
                t += 1
                (oh, orow), (gh, grow), _ = src.geometry(cfg)
                d_in = Dev(frame)
                d_out, d_orig = Dev(np.full((lanes, oh, orow), SENTINEL, np.uint8)), Dev(np.full((lanes, gh, grow), SENTINEL, np.uint8))
                src.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
                host_in = chain_submit.host_buffer(frame.shape, which == "rgb", lib, keep, 0)
                host_in[...] = frame
                out = chain_submit.host_buffer((lanes, oh, orow), True, lib, keep, SENTINEL)
                orig = chain_submit.host_buffer((lanes, gh, grow), False, lib, keep, SENTINEL)
                src.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, orow, orig.ctypes.data, grow)
                outs, want = (out, orig), (d_out, d_orig)
            else:
                frames = cs.clip(t, 3)
                t += 3
                cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
                cv = CanvasRgb(PLANAR_C if i % 8 == 0 else RGB_C, cw, chh, 3 * lanes, 2, 1)
                d_in = Dev(frames)
                cs.device_call(twin.magnifier, cfg, d_in.ptr, 3, LR, cv.struct())
                host_in = chain_submit.host_buffer(frames.shape, i % 8 == 4, lib, keep, 0)
                host_in[...] = frames
                canvas, mc = compose_submit.host_canvas(cv, i % 8 == 0, lib, keep)
                cs.submit(sub, cfg, host_in.ctypes.data, 3, LR, mc)
                outs, want = (canvas,), (cv.dev,)
            twin.magnifier.sync()
            pending.append((outs, host_in, twin.magnifier.lane_produced(), tuple(d.numpy() for d in want)))
            if len(pending) == 3 or i < 3:
                got, _, lp, exp = pending.pop(0)
                sub.magnifier.collect()
                assert np.array_equal(sub.magnifier.lane_produced(), lp)
                assert all(np.array_equal(g, e) for g, e in zip(got, exp)), i
        while pending:
            got, _, lp, exp = pending.pop(0)
            sub.magnifier.collect()
            assert np.array_equal(sub.magnifier.lane_produced(), lp)
            assert all(np.array_equal(g, e) for g, e in zip(got, exp))
        assert yuv420p.blobs(sub) == yuv420p.blobs(twin)
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)


# ---- errors ----------------------------------------------------------------------------------------------------------

def test_errors_return_before_any_launch_or_copy():
    """Every bad call is MC_ERR_INVALID with the launch count, every output, the canvases, the lanes' state (blobs) and
    the frames in flight unchanged"""
    w, h, lanes = 130, 74, 2
    cfg = chain_cfg(O.MODE_LAPLACE, MODES["laplace"][1], down=2)
    lay = Rgb(w, h, PLANAR, pitch=w + 2)
    xs = np.stack([from_bgr(lane_frame(0, k, w, h, 3), PLANAR) for k in range(lanes)])
    d_in = Dev(lay.pack(xs))
    lib, p = capi.lib(), _to_mc(cfg)
    ch = L.ProcessingChainB200(0, lanes=lanes)
    rgb_device_call(ch, cfg, xs, 1, lay)   # state to keep
    m = ch.magnifier
    before, n0 = yuv420p.blobs(ch), m.launch_count
    out_step, orig_step = 3 * (w // 2), 3 * (w // 2)
    d_out, d_orig = Dev(np.full((2 * lanes, h // 2, out_step), SENTINEL, np.uint8)), Dev(np.full((2 * lanes, h // 2, orig_step), SENTINEL, np.uint8))
    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
    cv = CanvasRgb(PLANAR_C, cw, chh, 2 * lanes, 2)
    rcv = CanvasRgb(RGB_C, cw, chh, 2 * lanes, 2)
    packed = Rgb(w, h, RGBA, pitch=4 * w)
    good = lay.struct(d_in.ptr)
    flags = np.zeros((2, lanes), np.uint8)
    base = dict(rp=good, frames=1, w=w, h=h, d_out=d_out.ptr, out_step=out_step, d_orig=d_orig.ptr, orig_step=orig_step,
                flags=flags, canvas=cv.struct(), split=LR)
    bad = [dict(rp=None), dict(rp=lay.struct(d_in.ptr, data=None)), dict(rp=lay.struct(d_in.ptr, g=None)),
           dict(rp=lay.struct(d_in.ptr, b=None)), dict(rp=lay.struct(d_in.ptr, layout=4)), dict(rp=lay.struct(d_in.ptr, layout=-1)),
           dict(w=0), dict(h=0), dict(w=-3), dict(rp=lay.struct(d_in.ptr, pitch=w - 1)),
           dict(rp=packed.struct(d_in.ptr, pitch=4 * w - 1)), dict(rp=packed.struct(d_in.ptr, layout=RGB, pitch=3 * w - 1)),
           dict(rp=lay.struct(d_in.ptr, lane_stride=(w + 2) * h - 1)), dict(frames=0), dict(frames=capi.MC_MAX_LANES),
           dict(flags=None), dict(out_step=out_step - 1), dict(orig_step=orig_step - 1), dict(d_out=None), dict(split=3),
           dict(canvas=cv.struct(data=None)), dict(canvas=cv.struct(pitch=cw - 1)),
           dict(canvas=cv.struct(lane_stride=3 * cv.pitch * chh - 1)), dict(canvas=rcv.struct(pitch=3 * cw - 1)),
           dict(canvas=rcv.struct(lane_stride=rcv.pitch * chh - 1)), dict(canvas=cv.struct(format=5))]
    compose_only = ("split", "canvas")
    for bd in bad:
        args = {**base, **bd}
        info = capi.McChainInfo()
        rp = C.byref(args["rp"]) if args["rp"] is not None else None
        u8 = args["flags"].ctypes.data_as(C.POINTER(C.c_uint8)) if args["flags"] is not None else None
        if not any(k in bd for k in compose_only):
            assert lib.mc_chain_process_rgb_device(m._h, rp, args["frames"], args["w"], args["h"], C.byref(p), 0,
                                                   args["d_out"], args["out_step"], args["d_orig"], args["orig_step"], u8,
                                                   C.byref(info)) == capi.MC_ERR_INVALID, bd
        if not any(k in bd for k in ("out_step", "orig_step", "d_out")):
            assert lib.mc_chain_compose_rgb_device(m._h, rp, args["frames"], args["w"], args["h"], C.byref(p), 0,
                                                   args["split"], C.byref(args["canvas"]), u8,
                                                   C.byref(info)) == capi.MC_ERR_INVALID, bd
    # a planar RGB canvas with a short lane stride, from a BGR source (the canvas error of every compose call)
    d_bgr = Dev(np.stack([lane_frame(0, k, w, h, 3) for k in range(lanes)]))
    assert lib.mc_chain_compose_device(m._h, d_bgr.ptr, 1, w, h, 3, 3 * w, C.byref(p), 0, LR,
                                       C.byref(cv.struct(lane_stride=cv.pitch * chh)), flags.ctypes.data_as(C.POINTER(C.c_uint8)),
                                       C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    m.sync()
    assert m.launch_count == n0
    assert (d_out.numpy() == SENTINEL).all() and (d_orig.numpy() == SENTINEL).all()
    assert (cv.dev.numpy() == SENTINEL).all() and (rcv.dev.numpy() == SENTINEL).all()
    assert yuv420p.blobs(ch) == before

    # the submits: every argument error before any copy, with a clip in flight left as it was
    m.set_option("pipeline_depth", 2)
    host = lay.pack(xs)
    hgood = lay.struct(host.ctypes.data)
    hcv = CanvasRgb(PLANAR_C, cw, chh, lanes, 2)
    hbuf, hmc = compose_submit.host_canvas(hcv, False, lib, [])
    prod = np.zeros(lanes, np.uint8)
    _, fl0 = ch.compose_submit_rgb(hgood, 1, w, h, cfg, LR, hmc)
    n1 = m.launch_count
    spare = np.full((lanes, h // 2, orig_step), SENTINEL, np.uint8)
    sub_bad = [None, lay.struct(host.ctypes.data, b=None), lay.struct(host.ctypes.data, layout=7),
               lay.struct(host.ctypes.data, pitch=w - 1), lay.struct(host.ctypes.data, lane_stride=1)]
    for rp in sub_bad:
        ref = C.byref(rp) if rp is not None else None
        assert lib.mc_chain_submit_rgb(m._h, ref, w, h, C.byref(p), 0, spare.ctypes.data, orig_step, None, 0,
                                       C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
        assert lib.mc_chain_compose_submit_rgb(m._h, ref, 1, w, h, C.byref(p), 0, LR, C.byref(hmc),
                                               prod.ctypes.data_as(C.POINTER(C.c_uint8)),
                                               C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert lib.mc_chain_compose_submit_rgb(m._h, C.byref(hgood), 1, w, h, C.byref(p), 0, LR,
                                           C.byref(capi.McCanvas(PLANAR_C, hmc.data, None, cw - 1, hmc.lane_stride)),
                                           prod.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert m.launch_count == n1 and (spare == SENTINEL).all() and (prod == 0).all()
    m.collect()
    # the collected clip is the device call's
    twin = L.ProcessingChainB200(0, lanes=lanes)
    rgb_device_call(twin, cfg, xs, 1, lay)
    tcv = CanvasRgb(PLANAR_C, cw, chh, lanes, 2)
    tfl, _ = compose_rgb(twin.magnifier, cfg, xs, 1, lay, LR, tcv)
    assert np.array_equal(fl0, tfl) and np.array_equal(hbuf, tcv.dev.numpy())


# ---- the exporter's shape against the compiled reference ----------------------------------------------------------------

@pytest.mark.skipif(EMU, reason="1080p clips of 16 on the CPU emulation take too long")
@pytest.mark.parametrize("layout,fmt", [(RGB, RGB_C), (BGRA, PLANAR_C)], ids=["rgb24_rgb", "bgra_planar"])
def test_1080p_export_with_labels_against_the_reference(layout, fmt):
    """2 lanes of 1080p frames, the benchmark's Laplace parameters (6 levels), a clip of 16 submitted with the exporter's
    labels, left/right into RGB canvases: lanes 0 and 1 within 1 LSB of the compiled reference fed cv2's conversion
    (the canvas built by compose(), the labels and the channel swap), and equal to the device compose call"""
    from compose_oracle import compose
    from common import make_cfgs, u8_diff
    from test_gpu_long_runs import RefCore
    w, h, n, lanes = 1920, 1080, 16, 2
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 6)
    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
    ov = export_labels(cw, chh, LR)
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    for ch in (sub, twin):
        ch.magnifier.set_overlay(ov)
    lay = Rgb(w, h, layout)
    xs = np.stack([from_bgr(lane_frame(t, k, w, h, 3), layout) for t in range(n) for k in range(lanes)])
    lib, keep = capi.lib(), []
    try:
        host_in = chain_submit.host_buffer((lay.block * n * lanes,), True, lib, keep, 0)
        host_in[...] = lay.pack(xs)
        cv = CanvasRgb(fmt, cw, chh, n * lanes)
        canvas, mc = compose_submit.host_canvas(cv, True, lib, keep)
        _, flags = sub.compose_submit_rgb(lay.struct(host_in.ctypes.data), n, w, h, cfg, LR, mc)
        sub.collect()
        tflags, _ = compose_rgb(twin.magnifier, cfg, xs, n, lay, LR, cv)
        assert flags.all() and np.array_equal(flags, tflags) and np.array_equal(canvas, cv.dev.numpy())
        seen_all = convert(xs, layout)
        for k in range(lanes):
            ref = RefCore(O.MODE_LAPLACE)
            for t in range(n):
                seen = seen_all[t * lanes + k]
                rprod, rout = ref.run(seen, ocfg)
                assert rprod, (k, t)
                got = np.full((max(cv.rows, 1), cv.pitch), SENTINEL, np.uint8)
                put_rgb(got, cv, ov.apply(compose(seen, rout, LR)))
                d = u8_diff(canvas[t * lanes + k], got)
                assert int(d.max()) <= 1, (k, t, int(d.max()))
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)
