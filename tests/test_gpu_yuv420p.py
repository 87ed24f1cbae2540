"""Planar 4:2:0 frames (I420 / YV12) into the chain and I420 export canvases: mc_chain_process_yuv420p_device,
mc_chain_compose_yuv420p_device, mc_chain_submit_yuv420p, mc_chain_compose_submit_yuv420p and MC_CANVAS_I420.

For any I420 input X a call must equal, bit for bit, the NV12 call on X with its chroma planes interleaved, and so the
BGR call on cv2.cvtColor(X, COLOR_YUV2BGR_I420): flags, info, lane flags, processed frames, original tap and the
temporal state, compared through mc_save_lane blobs (a save only reads; Color through its window taps).  Twin handles take the NV12 and the BGR calls.
An I420 canvas must be the NV12 canvas of the same call with its chroma de-interleaved; planes sit in sentinel-filled
buffers, so bytes written where they should not be (row padding between canvas_w / 2 and pitch / 2 included) show up."""
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
from test_gpu_chain_lanes import MODES, chain_cfg, device_call, info_tuple, none_cfg
from test_gpu_compose import Canvas
from test_gpu_lanes import SENTINEL, lane_frame, state_names
from test_gpu_nv12 import Dev, Layout
from test_gpu_yuv422 import Yuv, from_bgr, yuv_device_call

pytestmark = pytest.mark.gpu

EMU = os.environ.get("MC_EMU") == "1"
I420, NV12, BGR = capi.MC_CANVAS_I420, capi.MC_CANVAS_NV12, capi.MC_CANVAS_BGR
NONE, LR, TB = capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM


# ---- I420 frames and buffers ----------------------------------------------------------------------------------------

def to_i420(bgr):
    """BGR [h][w][3] -> cv2's I420 [3h/2][w] (Y, then the Cb plane, then the Cr plane)"""
    return cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)


def split_planes(x, h, w):
    """cv2's I420 [3h/2][w] -> (Y [h][w], Cb [h/2][w/2], Cr [h/2][w/2])"""
    f, n = x.ravel(), w * h
    return f[:n].reshape(h, w), f[n:n + n // 4].reshape(h // 2, w // 2), f[n + n // 4:].reshape(h // 2, w // 2)


def i420_to_nv12(x, h, w):
    """the NV12 frame of X's Y plane and its Cb, Cr planes interleaved: [3h/2][w]"""
    y, u, v = split_planes(x, h, w)
    return np.concatenate([y, np.stack([u, v], -1).reshape(h // 2, w)])


def i420_to_bgr(x, yv12=False):
    return cv2.cvtColor(x, cv2.COLOR_YUV2BGR_YV12 if yv12 else cv2.COLOR_YUV2BGR_I420)


class Lay:
    """Where an I420 frame set's three planes sit in one buffer of lanes blocks of `block` bytes, `offset` bytes from the
    buffer's start: arrangement "yuv" (each plane after the one before, with `gap` bytes between), "uvy" (the chroma
    planes before the luma plane) or "far" (the chroma planes a long way after the luma plane).  yv12: the buffer holds
    the Cr plane where I420 holds the Cb plane (the call is given u / v at the Cb / Cr planes)."""

    def __init__(self, w, h, pitch=None, chroma_pitch=None, arrangement="yuv", gap=0, offset=0, yv12=False):
        self.w, self.h, self.yv12 = w, h, yv12
        self.pitch = pitch or w
        self.cpitch = chroma_pitch or self.pitch // 2
        assert self.pitch >= w and self.cpitch >= w // 2
        ysz, csz = self.pitch * h, self.cpitch * (h // 2)
        if arrangement == "yuv":
            self.ofs = (0, ysz + gap, ysz + csz + 2 * gap)
        elif arrangement == "uvy":
            self.ofs = (2 * csz + 2 * gap, 0, csz + gap)
        else:
            self.ofs = (0, ysz + 4096 + gap, ysz + 4096 + csz + 3 * gap + 64)
        self.block = max(o + s for o, s in zip(self.ofs, (ysz, csz, csz))) + gap
        self.offset = offset

    @property
    def lane_stride(self):
        return self.block

    def pack(self, xs, fill=0x3C):
        buf = np.full(len(xs) * self.block + self.offset, fill, np.uint8)
        w, h = self.w, self.h
        for v, x in enumerate(xs):
            y, u, cr = split_planes(x, h, w)
            if self.yv12:
                u, cr = cr, u
            for (o, p, rows, row), plane in zip(((self.ofs[0], self.pitch, h, w), (self.ofs[1], self.cpitch, h // 2, w // 2),
                                                  (self.ofs[2], self.cpitch, h // 2, w // 2)), (y, u, cr)):
                base = self.offset + v * self.block + o
                buf[base:base + rows * p].reshape(rows, p)[:, :row] = plane
        return buf

    def struct(self, base, **override):
        y, u, v = (base + self.offset + o for o in self.ofs)
        if self.yv12:
            u, v = v, u
        f = dict(y=y, u=u, v=v, pitch=self.pitch, chroma_pitch=self.cpitch, lane_stride=self.block)
        f.update(override)
        return capi.McYuv420p(f["y"], f["u"], f["v"], f["pitch"], f["chroma_pitch"], f["lane_stride"])


class Canvas420(Canvas):
    """Canvas with MC_CANVAS_I420 as well: the luma plane, `uv_gap` rows, then the Cb plane and right after it the Cr
    plane, canvas_h / 2 rows of pitch / 2 bytes each (pitch = cw + pad, pad even)."""

    def __init__(self, fmt, cw, ch, v, pad=0, lane_rows=0, uv_gap=0):
        if fmt != I420:
            return super().__init__(fmt, cw, ch, v, pad, lane_rows, uv_gap)
        pad += pad % 2
        self.fmt, self.cw, self.ch = fmt, cw, ch
        self.pitch, self.uv_row = cw + pad, ch + uv_gap
        self.rows = self.uv_row + ch // 2 + lane_rows   # two chroma planes of ch / 2 rows of pitch / 2 bytes
        self.dev = Dev(np.full((v, max(self.rows, 1), max(self.pitch, 1)), SENTINEL, np.uint8))

    def expected(self, canvases):
        if self.fmt != I420:
            return super().expected(canvases)
        want = np.full((len(canvases), max(self.rows, 1), max(self.pitch, 1)), SENTINEL, np.uint8)
        for v, im in enumerate(canvases):
            if im is not None:
                put_i420(want[v], self, to_i420(np.ascontiguousarray(im)))
        return want


def put_i420(lane, cv, x):
    """cv2's I420 x of a cw x ch canvas into one lane [rows][pitch] of Canvas420 cv's layout"""
    y, u, v = split_planes(x, cv.ch, cv.cw)
    flat = lane.reshape(-1)
    flat.reshape(lane.shape)[:cv.ch, :cv.cw] = y
    half, base = cv.pitch // 2, cv.uv_row * cv.pitch
    for k, plane in enumerate((u, v)):
        o = base + k * half * (cv.ch // 2)
        flat[o:o + half * (cv.ch // 2)].reshape(cv.ch // 2, half)[:, :cv.cw // 2] = plane


def deinterleave(nv_lanes, nv_cv, cv, written):
    """the I420 buffer of Canvas420 cv that holds NV12 canvas nv_cv's lanes (nv_lanes) de-interleaved, for the lanes
    written; sentinel elsewhere"""
    want = np.full((len(written), max(cv.rows, 1), max(cv.pitch, 1)), SENTINEL, np.uint8)
    for v, wr in enumerate(written):
        if wr and cv.cw:
            y = nv_lanes[v, :cv.ch, :cv.cw]
            uv = nv_lanes[v, nv_cv.uv_row:nv_cv.uv_row + cv.ch // 2, :cv.cw]
            put_i420(want[v], cv, np.concatenate([y.ravel(), uv[:, 0::2].ravel(), uv[:, 1::2].ravel()]).reshape(-1, cv.cw))
    return want


def blobs(ch):
    return [ch.save_lane(k) for k in range(ch.lanes)]


def assert_same_state(a, b, mode):
    """Laplace and Phase: every lane's mc_save_lane blob.  Color: the window's read-only taps (a Color blob also carries
    the ring slots no frame has filled yet, whose bytes are whatever the allocation held)."""
    if mode == O.MODE_COLOR:
        for name, level in state_names(b.magnifier, mode):
            assert np.array_equal(a.magnifier.get_state(name, level), b.magnifier.get_state(name, level)), (name, level)
    elif mode != O.MODE_NONE:
        assert blobs(a) == blobs(b)


# ---- the chain against its NV12 and BGR twins -------------------------------------------------------------------------

def i420_call(ch, cfg, xs, frames, lay, out_pad=0, orig_pad=0, want_orig=True):
    """one mc_chain_process_yuv420p_device call on I420 frames xs [V][3h/2][w] -> (flags, info, out, orig)"""
    w, h = lay.w, lay.h
    g = ch.geometry(cfg, w, h, 3)
    out = (h, 3 * w) if g.cur_is_input else (g.out_h, g.out_w * g.out_channels)
    orig = (h, 3 * w) if g.orig_is_input else (g.orig_h, g.orig_w * 3)
    v = len(xs)
    d_in = Dev(lay.pack(xs))
    d_out = Dev(np.full((v, out[0], out[1] + out_pad), SENTINEL, np.uint8))
    d_orig = Dev(np.full((v, orig[0], orig[1] + orig_pad), SENTINEL, np.uint8)) if want_orig else None
    flags, info = ch.process_yuv420p_device(lay.struct(d_in.ptr), frames, w, h, cfg, d_out.ptr, out[1] + out_pad,
                                            d_orig.ptr if d_orig else 0, orig[1] + orig_pad)
    ch.magnifier.sync()
    return flags.astype(np.uint8), info, d_out.numpy(), d_orig.numpy() if d_orig else None


def check_420(mode, ui, w, h, steps, lanes=1, lay_kw=None, bgr_twin=True, color_lifecycle=False):
    """Handle A takes I420 calls, B the NV12 calls on the same frames, C the BGR calls on cv2's conversion.  steps:
    ("frame",) / ("clip", n); ("nv12",) / ("bgr",) / ("yuyv",) that call on every handle; ("restart", k) / ("hold", k, on) /
    ("lp", k) (lane k's amplification changed) on every handle; ("cfg", kwargs) chain settings."""
    cfg = chain_cfg(mode, ui)
    chains = [L.ProcessingChainB200(0, lanes=lanes) for _ in range(3 if bgr_twin else 2)]
    if color_lifecycle:
        for ch in chains:
            ch.magnifier.set_option("color_lane_lifecycle", 1)
    a, b = chains[0], chains[1]
    lay = Lay(w, h, **(lay_kw or {}))
    nv = Layout(w, h)
    t = 0
    for step in steps:
        if step[0] in ("restart", "hold", "lp"):
            for ch in chains:
                if step[0] == "restart":
                    ch.magnifier.restart_lane(step[1])
                elif step[0] == "hold":
                    ch.magnifier.hold_lane(step[1], step[2])
                else:
                    ch.set_lane_params(step[1], dataclasses.replace(cfg.magnification, amplification=cfg.magnification.amplification + 7))
            continue
        if step[0] == "cfg":
            cfg = chain_cfg(mode, ui, **step[1])
            continue
        n = step[1] if step[0] == "clip" else 1
        bgr = np.stack([lane_frame(s, k, w, h, 3) for s in range(t, t + n) for k in range(lanes)])
        t += n
        xs = np.stack([to_i420(f) for f in bgr])
        nvs = np.stack([i420_to_nv12(x, h, w) for x in xs])
        seen = np.stack([i420_to_bgr(x) for x in xs])
        if step[0] in ("nv12", "bgr", "yuyv"):
            rs = []
            for ch in chains:
                if step[0] == "nv12":
                    rs.append(device_call(ch, cfg, nvs, n, w, h, 3, nv12=nv))
                elif step[0] == "bgr":
                    rs.append(device_call(ch, cfg, seen, n, w, h, 3))
                else:
                    yx = np.stack([from_bgr(f, capi.MC_YUV422_YUYV) for f in seen])
                    rs.append(yuv_device_call(ch, cfg, yx, n, Yuv(w, h, capi.MC_YUV422_YUYV)))
            for r in rs[1:]:
                assert np.array_equal(r[0], rs[0][0]) and info_tuple(r[1]) == info_tuple(rs[0][1]), step
                assert np.array_equal(r[2], rs[0][2]) and np.array_equal(r[3], rs[0][3]), step
            continue
        ra = i420_call(a, cfg, xs, n, lay, 3, 5)
        rb = device_call(b, cfg, nvs, n, w, h, 3, nv12=nv, out_pad=3, orig_pad=5)
        twins = [rb] + ([device_call(chains[2], cfg, seen, n, w, h, 3, out_pad=3, orig_pad=5)] if bgr_twin else [])
        for r in twins:
            assert np.array_equal(ra[0], r[0]), (step, ra[0], r[0])
            assert info_tuple(ra[1]) == info_tuple(r[1]), (step, info_tuple(ra[1]), info_tuple(r[1]))
            assert np.array_equal(ra[2], r[2]), (step, np.argwhere(ra[2] != r[2])[:5])
            assert np.array_equal(ra[3], r[3]), step
        for ch in chains[1:]:
            assert np.array_equal(a.magnifier.lane_produced(), ch.magnifier.lane_produced()), step
    for ch in chains[1:]:
        assert_same_state(a, ch, mode)
    return a


def every_triple(w, h):
    """-> I420 [3h/2][w]: 2x2 block b carries the pair (Cb, Cr) = (b >> 8 & 255, b & 255) of b % 2^16 and the lumas 4r ..
    4r + 3 of its repetition r = b >> 16, so a 4096 x 4096 frame holds every (Y, Cb, Cr) triple once"""
    b = np.arange((w // 2) * (h // 2), dtype=np.uint32).reshape(h // 2, w // 2)
    pair, r = b & 0xFFFF, (b >> 16) & 63
    y = np.empty((h, w), np.uint8)
    for dy in (0, 1):
        for dx in (0, 1):
            y[dy::2, dx::2] = 4 * r + 2 * dy + dx
    return np.concatenate([y.ravel(), (pair >> 8).astype(np.uint8).ravel(), (pair & 255).astype(np.uint8).ravel()]).reshape(-1, w)


@pytest.mark.skipif(EMU, reason="every triple is too slow for the CPU emulation")
@pytest.mark.parametrize("yv12", [False, True], ids=["i420", "yv12"])
@pytest.mark.parametrize("w,h,lay_kw", [
    (4096, 4096, dict()),                                                    # tight planes, chroma_pitch = pitch / 2
    (4096, 4096, dict(pitch=4160, chroma_pitch=2050, arrangement="uvy")),   # chroma first, chroma_pitch unrelated
    (4090, 4096, dict(pitch=4096, chroma_pitch=2048, arrangement="far", gap=3, offset=1)),   # w = 2 mod 8, odd addresses
], ids=["tight", "chroma_first", "far_odd"])
def test_front_and_compose_on_every_triple(yv12, w, h, lay_kw):
    """Mode None with a full-frame ROI and grayscale: d_original is cv2's conversion and d_out its gray (the front), and
    an MC_SPLIT_NONE BGR canvas is the conversion too (the compose kernel's pane read).  YV12 is the same frame with its
    chroma planes swapped in memory and the call's u / v pointing at its Cb / Cr planes."""
    x = every_triple(w, h)
    want = i420_to_bgr(x)
    if yv12:
        y, u, v = split_planes(x, h, w)
        assert np.array_equal(i420_to_bgr(np.concatenate([y.ravel(), v.ravel(), u.ravel()]).reshape(-1, w), yv12=True), want)
    lay = Lay(w, h, yv12=yv12, **lay_kw)
    ch = L.ProcessingChainB200(0)
    flags, info, out, orig = i420_call(ch, none_cfg(roi=(0.0, 0.0, 1.0, 1.0), gray=True), x[None], 1, lay, 2, 6)
    assert not flags.any() and info_tuple(info) == (0, w, h, 1, 0, w, h, 3, 0)
    assert np.array_equal(orig[0][:, :3 * w], want.reshape(h, 3 * w)) and (orig[0][:, 3 * w:] == SENTINEL).all()
    assert np.array_equal(out[0][:, :w], cv2.cvtColor(want, cv2.COLOR_BGR2GRAY)) and (out[0][:, w:] == SENTINEL).all()
    cv = Canvas420(BGR, w, h, 1, pad=8)
    compose_420(ch.magnifier, none_cfg(), x[None], 1, lay, NONE, cv)
    assert np.array_equal(cv.dev.numpy(), cv.expected([want]))


W, H = (46, 30) if EMU else (134, 78)
FRONT_CASES = [dict(), dict(gray=True), dict(roi=(0.015, 0.013, 0.5, 0.8)), dict(down=2), dict(down=4, gray=True),
               dict(down=8), dict(down=3, roi=(0.1, 0.15, 0.8, 0.75))]   # ROI at an odd column and row; fractional area


@pytest.mark.parametrize("settings", FRONT_CASES, ids=["none", "gray", "roi_odd", "down2", "down4_gray", "down8", "roi_down3"])
@pytest.mark.parametrize("lay_kw", [dict(pitch=W + 10, chroma_pitch=W // 2 + 3, arrangement="uvy"),
                                    dict(pitch=W + 2, chroma_pitch=W // 2 + 1, arrangement="far", offset=1, gap=1)],
                         ids=["vec", "bytes"])
def test_front_matches_the_nv12_front(settings, lay_kw):
    """Mode None over 3 lanes x 2 frames: the front's tap walk on I420 equals it on NV12 and on cv2's BGR"""
    check_420(O.MODE_NONE, MODES["laplace"][1], W, H, [("cfg", settings), ("clip", 2), ("frame",)], lanes=3, lay_kw=lay_kw)


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("settings", [dict(), dict(gray=True), dict(down=2), dict(roi=(0.015, 0.013, 0.6, 0.8))],
                         ids=["none", "gray", "down2", "roi_odd"])
@pytest.mark.parametrize("lanes", [1, 3])
def test_chain_equals_nv12_and_bgr_chains(mname, settings, lanes):
    """frames and clips of 1, 3 and 16; restart, hold and lane parameters on 3 lanes (Color with color_lane_lifecycle)"""
    mode, ui = MODES[mname]
    lifecycle = [] if lanes == 1 else [("restart", 2), ("hold", 1, 1), ("frame",), ("clip", 3), ("hold", 1, 0), ("lp", 0)]
    steps = [("cfg", settings), ("frame",), ("clip", 3), *lifecycle, ("clip", 16 if not EMU else 2), ("frame",), ("clip", 1)]
    check_420(mode, ui, W, H, steps, lanes=lanes, lay_kw=dict(pitch=W + 64), color_lifecycle=mname == "color")


@pytest.mark.parametrize("mname", list(MODES))
def test_i420_nv12_yuyv_and_bgr_calls_interleave(mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("nv12",), ("frame",), ("yuyv",), ("clip", 3), ("bgr",), ("frame",), ("cfg", dict(down=2)), ("frame",),
             ("nv12",), ("yuyv",), ("frame",)]
    check_420(mode, ui, W, H, steps, lanes=2, color_lifecycle=mname == "color")


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
@pytest.mark.parametrize("mname", list(MODES))
def test_1080p(mname):
    mode, ui = MODES[mname]
    check_420(mode, ui, 1920, 1080, [("frame",), ("frame",), ("clip", 3), ("frame",)], bgr_twin=False,
              lay_kw=dict(pitch=1920, chroma_pitch=960))


# ---- compose: I420 sources, and I420 canvases from every source -------------------------------------------------------

def compose_420(m, cfg, xs, n, lay, split, cv):
    d_in = Dev(lay.pack(xs))
    flags, info = m.chain_compose_yuv420p_device(lay.struct(d_in.ptr), n, lay.w, lay.h, cfg, split, cv.struct())
    m.sync()
    return flags.astype(np.uint8), info


def check_compose_420(mode, ui, w, h, fmt, split, steps, lanes=1, src="i420", labels=False, lay_kw=None, pad=6, lane_rows=1,
                      uv_gap=3):
    """Handle A composes `src` frames into `fmt` canvases; its twin B composes the NV12 frames of the same content into
    canvases of the same format (NV12 for an I420 canvas, which must then be B's de-interleaved).  src "i420": A takes
    I420 frames; "bgr" / "gray" / "nv12" / "yuyv": both take that source, and only the canvas format differs."""
    cfg = chain_cfg(mode, ui)
    a, b = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    lay, nv = Lay(w, h, **(lay_kw or {})), Layout(w, h, pitch=w + 4, uv_row=h + 2)
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
        cva = Canvas420(fmt, cw, chh, v, pad, lane_rows, uv_gap)
        cvb = Canvas420(NV12 if fmt == I420 else fmt, cw, chh, v, pad, lane_rows, uv_gap)
        xs = np.stack([to_i420(f) for f in bgr])
        nvs = np.stack([i420_to_nv12(x, h, w) for x in xs])
        if src in ("i420", "nv12"):
            ra = compose_420(a.magnifier, cfg, xs, n, lay, split, cva) if src == "i420" else None
            d_nv = Dev(nv.pack(nvs, fill=0x3C))
            if src == "nv12":
                ra = a.magnifier.chain_compose_nv12_device(nv.planes(d_nv.ptr), n, w, h, cfg, split, cva.struct())
            rb = b.magnifier.chain_compose_nv12_device(nv.planes(d_nv.ptr), n, w, h, cfg, split, cvb.struct())
        elif src == "yuyv":
            yl = Yuv(w, h, capi.MC_YUV422_YUYV, pitch=2 * w + 2)
            d_y = Dev(yl.pack(np.stack([from_bgr(f, capi.MC_YUV422_YUYV) for f in bgr])))
            ra = a.magnifier.chain_compose_yuv422_device(yl.struct(d_y.ptr), n, w, h, cfg, split, cva.struct())
            rb = b.magnifier.chain_compose_yuv422_device(yl.struct(d_y.ptr), n, w, h, cfg, split, cvb.struct())
        else:
            frames = bgr if c == 3 else np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr])
            d_in = Dev(frames)
            ra = a.magnifier.chain_compose_device(d_in.ptr, n, w, h, c, w * c, cfg, split, cva.struct())
            rb = b.magnifier.chain_compose_device(d_in.ptr, n, w, h, c, w * c, cfg, split, cvb.struct())
        a.magnifier.sync()
        b.magnifier.sync()
        assert np.array_equal(ra[0], rb[0]) and info_tuple(ra[1]) == info_tuple(rb[1]), step
        assert np.array_equal(a.magnifier.lane_produced(), b.magnifier.lane_produced())
        got, ref = cva.dev.numpy(), cvb.dev.numpy()
        if fmt == I420:
            ref = deinterleave(ref, cvb, cva, [not held[k % lanes] and cw > 0 for k in range(v)])
        assert np.array_equal(got, ref), (step, np.argwhere(got != ref)[:5])
    assert_same_state(a, b, mode)


SPLITS = {"none": NONE, "left_right": LR, "top_bottom": TB}


@pytest.mark.parametrize("fmt", [BGR, NV12, I420], ids=["bgr_canvas", "nv12_canvas", "i420_canvas"])
@pytest.mark.parametrize("split", list(SPLITS))
def test_i420_sources_into_every_canvas(split, fmt):
    steps = [("frame",), ("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 3), ("hold", 1, 1), ("cfg", dict(down=2)),
             ("frame",), ("hold", 1, 0), ("restart", 0), ("cfg", dict(gray=True)), ("clip", 2)]
    check_compose_420(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, SPLITS[split], steps, lanes=2, labels=split != "none",
                      lay_kw=dict(pitch=W + 2, chroma_pitch=W // 2 + 5, arrangement="far", offset=1))


@pytest.mark.parametrize("src", ["bgr", "gray", "nv12", "yuyv", "i420"])
@pytest.mark.parametrize("split", list(SPLITS))
def test_i420_canvas_from_every_source(src, split):
    """labels included; the canvas's row padding of all three planes stays sentinel"""
    steps = [("frame",), ("clip", 3), ("cfg", dict(down=2)), ("frame",)]
    check_compose_420(O.MODE_LAPLACE, MODES["laplace"][1], W, H, I420, SPLITS[split], steps, lanes=1, src=src, labels=True,
                      pad=10, lane_rows=2, uv_gap=1)


@pytest.mark.parametrize("mname", ["phase", "color"])
@pytest.mark.parametrize("aligned", [True, False], ids=["vec", "bytes"])
def test_i420_canvas_frames_not_produced(mname, aligned):
    """Phase's first frame and Color's warm-up compose the front's output; 8-byte aligned canvases or the byte path"""
    mode, ui = MODES[mname]
    steps = [("frame",), ("clip", 3), ("frame",)]
    pad, gap = (0, 0) if aligned else (6, 1)
    check_compose_420(mode, ui, 64, 32, I420, LR, steps, pad=pad, uv_gap=gap,
                      lay_kw=None if aligned else dict(pitch=66, chroma_pitch=35, offset=1))


def test_empty_i420_canvas_writes_nothing():
    """a 1 x 1 chain output has a 0 x 0 canvas: nothing is written"""
    cfg = chain_cfg(O.MODE_LAPLACE, MODES["laplace"][1], down=8)
    w, h = 14, 12
    assert L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR) == (0, 0)
    ch = L.ProcessingChainB200(0)
    cv = Canvas420(I420, 0, 0, 1)
    cv.dev = Dev(np.full((1, 4, 8), SENTINEL, np.uint8))
    x = to_i420(lane_frame(0, 0, w, h, 3))
    d_in = Dev(Lay(w, h).pack(x[None]))
    ch.magnifier.chain_compose_yuv420p_device(Lay(w, h).struct(d_in.ptr), 1, w, h, cfg, LR,
                                              capi.McCanvas(I420, cv.dev.ptr, cv.dev.ptr + 16, 2, 32))
    ch.magnifier.sync()
    assert (cv.dev.numpy() == SENTINEL).all()


# ---- submits: the pipelined checkers of the other sources, with I420 frames and canvases -----------------------------

class ChainSource(chain_submit.Source):
    def __init__(self, kind, lanes, w, h, pad):
        if kind != "i420":
            return super().__init__(kind, lanes, w, h, pad)
        self.kind, self.lanes, self.w, self.h, self.c = kind, lanes, w, h, 3
        self.lay = Lay(w, h, pitch=w + pad, chroma_pitch=w // 2 + pad // 2 + 1, arrangement="uvy" if pad else "yuv", gap=pad)

    def frame(self, t):
        if self.kind != "i420":
            return super().frame(t)
        return self.lay.pack(np.stack([to_i420(lane_frame(t, k, self.w, self.h, 3)) for k in range(self.lanes)]))

    def device_call(self, ch, cfg, d_in, d_out, out_step, d_orig, orig_step):
        if self.kind != "i420":
            return super().device_call(ch, cfg, d_in, d_out, out_step, d_orig, orig_step)
        return ch.process_yuv420p_device(self.lay.struct(d_in), 1, self.w, self.h, cfg, d_out, out_step, d_orig, orig_step)

    def submit(self, ch, cfg, base, out, out_step, orig, orig_step):
        if self.kind != "i420":
            return super().submit(ch, cfg, base, out, out_step, orig, orig_step)
        return ch.submit_yuv420p(self.lay.struct(base), self.w, self.h, cfg, out, out_step, orig, orig_step)


class ClipSource(compose_submit.ClipSource):
    def __init__(self, kind, lanes, w, h, pad):
        super().__init__("bgr" if kind == "i420" else kind, lanes, w, h, pad)
        if kind == "i420":
            self.kind = kind
            self.lay = Lay(w, h, pitch=w + pad, chroma_pitch=w // 2 + pad, arrangement="far" if pad else "yuv", gap=pad)

    def pack(self, bgr):
        if self.kind != "i420":
            return super().pack(bgr)
        return self.lay.pack(np.stack([to_i420(f) for f in bgr]))

    def device_call(self, m, cfg, d_in, n, split, canvas):
        if self.kind != "i420":
            return super().device_call(m, cfg, d_in, n, split, canvas)
        return m.chain_compose_yuv420p_device(self.lay.struct(d_in), n, self.w, self.h, cfg, split, canvas)

    def submit(self, ch, cfg, base, n, split, canvas):
        if self.kind != "i420":
            return super().submit(ch, cfg, base, n, split, canvas)
        return ch.compose_submit_yuv420p(self.lay.struct(base), n, self.w, self.h, cfg, split, canvas)


@pytest.fixture()
def i420_submits(monkeypatch):
    """the submit checkers of test_gpu_chain_submit / test_gpu_compose_submit, with the "i420" source and I420 canvases"""
    monkeypatch.setattr(chain_submit, "Source", ChainSource)
    monkeypatch.setattr(compose_submit, "ClipSource", ClipSource)
    monkeypatch.setattr(compose_submit, "Canvas", Canvas420)


@pytest.mark.parametrize("front", ["none", "roi", "down2", "gray", "roi_down_gray"])
@pytest.mark.parametrize("depth", [1, 3, 5])
def test_chain_submit_equals_the_device_chain(i420_submits, front, depth):
    """restarts, holds, an amplification change, a ROI move and a levels change in flight; pinned and pageable planes"""
    pins = [(True, False, True), (False, True, False), (True, True, True)][depth // 2]
    chain_submit.check_chain_submit("i420", front, "laplace", lanes=3, depth=depth, pins=pins, n=14 if EMU else 20)


@pytest.mark.parametrize("kind,fmt,split", [("i420", I420, LR), ("i420", BGR, TB), ("i420", NV12, NONE), ("bgr", I420, TB),
                                            ("nv12", I420, NONE), ("yuyv", I420, LR), ("gray", I420, LR)])
@pytest.mark.parametrize("depth", [1, 3, 5])
def test_compose_submit_equals_the_device_compose(i420_submits, kind, fmt, split, depth):
    """clips of 16, 3 and 1 and a shorter last clip; an overlay set / replaced / cleared, restarts, holds, lane params, a ROI
    move and a levels change in flight; input and canvas pinned and pageable in turn"""
    clips = (4, 3, 1, 4, 2) if EMU else compose_submit.CLIPS
    compose_submit.check_compose_submit(kind, "roi" if depth != 3 else "down2", "laplace", lanes=2, depth=depth, clips=clips,
                                        fmt=fmt, split=split, pad=6)


@pytest.mark.parametrize("mname", ["phase", "color"])
def test_compose_submit_modes(i420_submits, mname):
    compose_submit.check_compose_submit("i420", "gray", mname, lanes=3, depth=3, clips=(3, 2, 1, 3), fmt=I420, split=LR)


def test_submits_interleave_in_fifo_order_with_nv12_and_yuyv(i420_submits):
    """mc_chain_compose_submit_yuv420p, mc_submit_nv12 and mc_chain_submit_yuv422 in turn on one handle, each collect
    equal to its own device call on a twin that runs them in the same order"""
    w, h, lanes = W, H, 2
    cfg = chain_cfg(*MODES["laplace"])
    sub, twin = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    yv, cs = ChainSource("yuyv", lanes, w, h, 4), ClipSource("i420", lanes, w, h, 2)
    nvl = Layout(w, h, pitch=w + 2, uv_row=h + 1)
    lib, keep, pending, t = capi.lib(), [], [], 0
    try:
        for i in range(9):
            which = ("compose", "nv12", "yuyv")[i % 3]
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
            elif which == "yuyv":
                frame = yv.frame(t)
                t += 1
                (oh, orow), (gh, grow), _ = yv.geometry(cfg)
                d_in = Dev(frame)
                d_out, d_orig = Dev(np.full((lanes, oh, orow), SENTINEL, np.uint8)), Dev(np.full((lanes, gh, grow), SENTINEL, np.uint8))
                yv.device_call(twin, cfg, d_in.ptr, d_out.ptr, orow, d_orig.ptr, grow)
                host_in = chain_submit.host_buffer(frame.shape, False, lib, keep, 0)
                host_in[...] = frame
                out = chain_submit.host_buffer((lanes, oh, orow), True, lib, keep, SENTINEL)
                orig = chain_submit.host_buffer((lanes, gh, grow), False, lib, keep, SENTINEL)
                yv.submit(sub, cfg, host_in.ctypes.data, out.ctypes.data, orow, orig.ctypes.data, grow)
                outs, want = (out, orig), (d_out, d_orig)
            else:
                frames = cs.clip(t, 3)
                t += 3
                cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
                cv = Canvas420(I420, cw, chh, 3 * lanes, 2, 1, 2)
                d_in = Dev(frames)
                cs.device_call(twin.magnifier, cfg, d_in.ptr, 3, LR, cv.struct())
                host_in = chain_submit.host_buffer(frames.shape, i % 2 == 1, lib, keep, 0)
                host_in[...] = frames
                canvas, mc = compose_submit.host_canvas(cv, i % 2 == 0, lib, keep)
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
        assert blobs(sub) == blobs(twin)
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
    lay = Lay(w, h, pitch=w + 2)
    xs = np.stack([to_i420(lane_frame(0, k, w, h, 3)) for k in range(lanes)])
    d_in = Dev(lay.pack(xs))
    lib, p = capi.lib(), _to_mc(cfg)
    ch = L.ProcessingChainB200(0, lanes=lanes)
    i420_call(ch, cfg, xs, 1, lay)   # state to keep
    m = ch.magnifier
    before, n0 = blobs(ch), m.launch_count
    out_step, orig_step = w // 2, 3 * (w // 2)
    d_out, d_orig = Dev(np.full((2 * lanes, h // 2, out_step), SENTINEL, np.uint8)), Dev(np.full((2 * lanes, h // 2, orig_step), SENTINEL, np.uint8))
    cw, chh = L.MagnificationProcessor.compose_geometry(cfg, w, h, 3, LR)
    cv = Canvas420(I420, cw, chh, 2 * lanes, 2)
    good = lay.struct(d_in.ptr)
    flags = np.zeros((2, lanes), np.uint8)
    base = dict(yp=good, frames=1, w=w, h=h, d_out=d_out.ptr, out_step=out_step, d_orig=d_orig.ptr, orig_step=orig_step,
                flags=flags, canvas=cv.struct(), split=LR)
    bad = [dict(yp=None), dict(yp=lay.struct(d_in.ptr, y=None)), dict(yp=lay.struct(d_in.ptr, u=None)),
           dict(yp=lay.struct(d_in.ptr, v=None)), dict(w=w - 1), dict(h=h - 1), dict(w=0), dict(h=0),
           dict(yp=lay.struct(d_in.ptr, pitch=w - 1)), dict(yp=lay.struct(d_in.ptr, chroma_pitch=w // 2 - 1)),
           dict(yp=lay.struct(d_in.ptr, lane_stride=(w + 2) * h - 1)), dict(frames=0), dict(frames=capi.MC_MAX_LANES),
           dict(flags=None), dict(out_step=out_step - 1), dict(orig_step=orig_step - 1), dict(d_out=None), dict(split=3),
           dict(canvas=cv.struct(data=None)), dict(canvas=cv.struct(uv=None)), dict(canvas=cv.struct(pitch=cv.pitch + 1)),
           dict(canvas=cv.struct(pitch=cw - 2)), dict(canvas=cv.struct(lane_stride=1)), dict(canvas=cv.struct(format=3))]
    compose_only = ("split", "canvas")
    for bd in bad:
        args = {**base, **bd}
        info = capi.McChainInfo()
        yp = C.byref(args["yp"]) if args["yp"] is not None else None
        u8 = args["flags"].ctypes.data_as(C.POINTER(C.c_uint8)) if args["flags"] is not None else None
        if not any(k in bd for k in compose_only):
            assert lib.mc_chain_process_yuv420p_device(m._h, yp, args["frames"], args["w"], args["h"], C.byref(p), 0,
                                                       args["d_out"], args["out_step"], args["d_orig"], args["orig_step"], u8,
                                                       C.byref(info)) == capi.MC_ERR_INVALID, bd
        if not any(k in bd for k in ("out_step", "orig_step", "d_out")):
            assert lib.mc_chain_compose_yuv420p_device(m._h, yp, args["frames"], args["w"], args["h"], C.byref(p), 0,
                                                       args["split"], C.byref(args["canvas"]), u8,
                                                       C.byref(info)) == capi.MC_ERR_INVALID, bd
    # an I420 canvas with a NULL uv, from a BGR source (the canvas error of every compose call)
    d_bgr = Dev(np.stack([lane_frame(0, k, w, h, 3) for k in range(lanes)]))
    assert lib.mc_chain_compose_device(m._h, d_bgr.ptr, 1, w, h, 3, 3 * w, C.byref(p), 0, LR, C.byref(cv.struct(uv=None)),
                                       flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    m.sync()
    assert m.launch_count == n0
    assert (d_out.numpy() == SENTINEL).all() and (d_orig.numpy() == SENTINEL).all() and (cv.dev.numpy() == SENTINEL).all()
    assert blobs(ch) == before

    # the submits: every argument error before any copy, with a clip in flight left as it was
    m.set_option("pipeline_depth", 2)
    host = lay.pack(xs)
    hgood = lay.struct(host.ctypes.data)
    hcv = Canvas420(I420, cw, chh, lanes, 2)
    hbuf, hmc = compose_submit.host_canvas(hcv, False, lib, [])
    prod = np.zeros(lanes, np.uint8)
    _, fl0 = ch.compose_submit_yuv420p(hgood, 1, w, h, cfg, LR, hmc)
    n1 = m.launch_count
    spare = np.full((lanes, h // 2, orig_step), SENTINEL, np.uint8)
    sub_bad = [None, lay.struct(host.ctypes.data, u=None), lay.struct(host.ctypes.data, chroma_pitch=w // 2 - 1),
               lay.struct(host.ctypes.data, lane_stride=1)]
    for yp in sub_bad:
        ref = C.byref(yp) if yp is not None else None
        assert lib.mc_chain_submit_yuv420p(m._h, ref, w, h, C.byref(p), 0, spare.ctypes.data, orig_step, None, 0,
                                           C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
        assert lib.mc_chain_compose_submit_yuv420p(m._h, ref, 1, w, h, C.byref(p), 0, LR, C.byref(hmc),
                                                   prod.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                   C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert lib.mc_chain_compose_submit_yuv420p(m._h, C.byref(hgood), 1, w, h, C.byref(p), 0, LR,
                                               C.byref(capi.McCanvas(I420, hmc.data, hmc.uv, hmc.pitch + 1, hmc.lane_stride)),
                                               prod.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(capi.McChainInfo())) == capi.MC_ERR_INVALID
    assert m.launch_count == n1 and (spare == SENTINEL).all() and (prod == 0).all()
    m.collect()
    # the collected clip is the device call's
    twin = L.ProcessingChainB200(0, lanes=lanes)
    i420_call(twin, cfg, xs, 1, lay)
    tcv = Canvas420(I420, cw, chh, lanes, 2)
    tfl, _ = compose_420(twin.magnifier, cfg, xs, 1, lay, LR, tcv)
    assert np.array_equal(fl0, tfl) and np.array_equal(hbuf, tcv.dev.numpy())


# ---- the exporter's shape against the compiled reference ----------------------------------------------------------------

@pytest.mark.skipif(EMU, reason="1080p clips of 16 on the CPU emulation take too long")
def test_1080p_export_with_labels_against_the_reference():
    """2 lanes of 1080p I420, the benchmark's Laplace parameters (6 levels), a clip of 16 submitted with the exporter's
    labels, left/right into I420 canvases: lanes 0 and 1 within 1 LSB of the compiled reference fed cv2's conversion
    (the canvas built by compose(), the labels and cvtColor(BGR2YUV_I420)), and equal to the device compose call"""
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
    lay = Lay(w, h)
    xs = np.stack([to_i420(lane_frame(t, k, w, h, 3)) for t in range(n) for k in range(lanes)])
    lib, keep = capi.lib(), []
    try:
        host_in = chain_submit.host_buffer((lay.block * n * lanes,), True, lib, keep, 0)
        host_in[...] = lay.pack(xs)
        cv = Canvas420(I420, cw, chh, n * lanes)
        canvas, mc = compose_submit.host_canvas(cv, True, lib, keep)
        _, flags = sub.compose_submit_yuv420p(lay.struct(host_in.ctypes.data), n, w, h, cfg, LR, mc)
        sub.collect()
        tflags, _ = compose_420(twin.magnifier, cfg, xs, n, lay, LR, cv)
        assert flags.all() and np.array_equal(flags, tflags) and np.array_equal(canvas, cv.dev.numpy())
        for k in range(lanes):
            ref = RefCore(O.MODE_LAPLACE)
            for t in range(n):
                seen = i420_to_bgr(xs[t * lanes + k])
                rprod, rout = ref.run(seen, ocfg)
                assert rprod, (k, t)
                want = to_i420(ov.apply(compose(seen, rout, LR)))
                got = np.full((max(cv.rows, 1), cv.pitch), SENTINEL, np.uint8)
                put_i420(got, cv, want)
                d = u8_diff(canvas[t * lanes + k], got)
                assert int(d.max()) <= 1, (k, t, int(d.max()))
    finally:
        sub.magnifier.close()
        for p in keep:
            lib.mc_host_free(p)
