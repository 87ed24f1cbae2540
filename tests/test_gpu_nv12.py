"""NV12 frames in and out of the magnifier (mc_process_nv12_device / mc_process_clip_nv12_device / mc_submit_nv12).

For any NV12 input X an NV12 call must give, bit for bit, to_nv12(bgr_call(to_bgr(X))): to_bgr is cv2's
COLOR_YUV2BGR_NV12, to_nv12 cv2's COLOR_BGR2YUV_I420 with the chroma planes interleaved.  That covers the output bytes
(a lane or frame that did not produce leaves both planes untouched), the produced flags and the temporal state.  The
two conversion kernels are also checked alone, through the test hooks mc_debug_nv12_to_bgr / mc_debug_bgr_to_nv12,
against cv2 on every (Y, Cb, Cr) triple and every BGR colour."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_clip import assert_states_equal, run_clip
from test_gpu_lanes import LAPLACE_UI, PHASE_UI, COLOR_UI, SENTINEL, lane_frame, proc, process_raw

EMU = os.environ.get("MC_EMU") == "1"


# ---- conversions as cv2 does them, and NV12 buffers -----------------------------------------------------------------

def to_bgr(nv):
    """packed NV12 [3h/2][w] -> BGR [h][w][3]"""
    return cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12)


def to_nv12(bgr):
    """BGR [h][w][3] -> packed NV12 [3h/2][w]: cv2's I420 with Cb, Cr interleaved"""
    h, w = bgr.shape[:2]
    i420, n = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420).ravel(), w * h
    uv = np.stack([i420[n:n + n // 4], i420[n + n // 4:]], -1).reshape(h // 2, w)
    return np.concatenate([i420[:n].reshape(h, w), uv])


class Layout:
    """Where a frame set's planes sit in one buffer of `lanes` blocks of `rows` rows of `pitch` bytes: the luma plane at
    row 0 of a block, the Cb,Cr plane at row `uv_row` (h: packed frames; 1088 for a 1080p decoder surface)."""

    def __init__(self, w, h, pitch=None, uv_row=None, rows=None):
        self.w, self.h = w, h
        self.pitch = pitch or w
        self.uv_row = h if uv_row is None else uv_row
        self.rows = rows or self.uv_row + h // 2

    @property
    def lane_stride(self):
        return self.pitch * self.rows

    def pack(self, nv, fill=SENTINEL):
        """[V][3h/2][w] packed frames -> [V][rows][pitch] buffer (bytes outside the planes = fill)"""
        buf = np.full((len(nv), self.rows, self.pitch), fill, np.uint8)
        self.put(buf, range(len(nv)), nv)
        return buf

    def put(self, buf, lanes, nv):
        h, w = self.h, self.w
        for v, f in zip(lanes, nv):
            buf[v, :h, :w] = f[:h]
            buf[v, self.uv_row:self.uv_row + h // 2, :w] = f[h:]

    def planes(self, base):
        return capi.McNv12(base, base + self.uv_row * self.pitch, self.pitch, self.lane_stride)


class Dev:
    """A device copy of a host array (torch on the GPU; on the CUDA emulation device memory is host memory)."""

    def __init__(self, host):
        if EMU or "cuda_emu" in capi.LIB_PATH:
            self.a = np.ascontiguousarray(host).copy()
            self.ptr = self.a.ctypes.data
        else:
            import torch
            self.t = torch.from_numpy(np.ascontiguousarray(host)).cuda()
            torch.cuda.synchronize()
            self.ptr = self.t.data_ptr()

    def numpy(self):
        return self.a.copy() if hasattr(self, "a") else self.t.cpu().numpy()


# ---- the contract against the BGR path ------------------------------------------------------------------------------

def source(t, n, lanes, w, h, kind):
    """BGR [n][lanes][h][w][3] of frames t .. t+n-1: synthetic motion, or a full-range content kind"""
    if kind is None:
        return np.stack([np.stack([lane_frame(s, k, w, h, 3) for k in range(lanes)]) for s in range(t, t + n)])
    from test_gpu_full_range import content
    return np.stack([np.stack([content(kind, s, w, h, seed=k) for k in range(lanes)]) for s in range(t, t + n)])


def composition(p):
    return {k: v[0] for k, v in p.profile_read().items()}


def check_nv12(mode, ui, w, h, steps, lanes=1, options=(), layout=None, kind=None, launches=False):
    """Handle A takes NV12 calls, handle B (same options) the BGR calls on cv2's conversion of the same NV12 input.
    steps: ("frame",) / ("clip", n) NV12 calls on A; ("bgr",) a BGR frame call on both; ("restart", k) / ("hold", k, on)
    on both.  After every call A's NV12 buffer (sentinel-filled, padding included) must be B's output converted by cv2
    where B produced and the sentinel elsewhere, with the same flags; at the end the state planes are equal.  launches:
    A's kernels are B's plus nv12_to_bgr once and bgr_to_nv12 once (none when nothing produced).  -> A's flags per call."""
    cfg, _ = make_cfgs(mode, *ui)
    opts = tuple(options) + ((("profile_kernels", 1),) if launches else ())
    a, b = proc(lanes, opts), proc(lanes, opts)
    lay = layout or Layout(w, h)
    got, t = [], 0
    for step in steps:
        if step[0] in ("restart", "hold"):
            for p in (a, b):
                p.restart_lane(step[1]) if step[0] == "restart" else p.hold_lane(step[1], step[2])
            continue
        n = step[1] if step[0] == "clip" else 1
        src = source(t, n, lanes, w, h, kind)
        x = np.stack([to_nv12(f) for f in src.reshape(-1, h, w, 3)])
        bgr_in = np.stack([to_bgr(f) for f in x]).reshape(n, lanes, h, w, 3)
        t += n
        if step[0] == "bgr":
            pa, oa, fa = process_raw(a, bgr_in[0], cfg)
            pb, ob, fb = process_raw(b, bgr_in[0], cfg)
            assert pa == pb and np.array_equal(fa, fb) and np.array_equal(oa, ob)
            if launches:
                assert composition(a) == composition(b)
            continue
        if step[0] == "frame":
            _, ref, flags = process_raw(b, bgr_in[0], cfg)
            ref, flags = ref[None], flags[None].astype(np.uint8)
        else:
            flags, ref = run_clip(b, bgr_in, cfg)
        d_in, d_out = Dev(lay.pack(x, fill=0x3C)), Dev(np.full((n * lanes, lay.rows, lay.pitch), SENTINEL, np.uint8))
        if step[0] == "frame":
            produced = a.process_nv12_device(lay.planes(d_in.ptr), w, h, cfg, lay.planes(d_out.ptr))
            gflags = a.lane_produced()[None].astype(np.uint8)
            assert produced == bool(flags.any())
        else:
            gflags = a.process_clip_nv12_device(lay.planes(d_in.ptr), n, w, h, cfg, lay.planes(d_out.ptr)).astype(np.uint8)
        a.sync()
        assert np.array_equal(gflags, flags), (step, gflags, flags)
        assert np.array_equal(a.lane_produced(), b.lane_produced())
        want = np.full((n * lanes, lay.rows, lay.pitch), SENTINEL, np.uint8)
        vl = [v for v in range(n * lanes) if flags.ravel()[v]]
        lay.put(want, vl, [to_nv12(ref.reshape(-1, h, w, 3)[v]) for v in vl])
        assert np.array_equal(d_out.numpy(), want), step
        if launches:
            ca, cb = composition(a), composition(b)
            extra = {("nv12_to_bgr", 0): 1}
            if flags.any():
                extra[("bgr_to_nv12", 0)] = 1
            assert ca == {**cb, **extra}, (step, ca, cb)
        got.append(gflags)
    assert_states_equal(a, b, mode)
    a.close()
    b.close()
    return got


MODES = {"laplace": (O.MODE_LAPLACE, LAPLACE_UI), "phase": (O.MODE_PHASE, PHASE_UI), "color": (O.MODE_COLOR, COLOR_UI)}


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mname", list(MODES))
def test_frames_and_clips_equal_the_bgr_path(mname):
    """T = 1, 5, 16 on a fresh handle, then on the continuing one; frame calls before and after"""
    mode, ui = MODES[mname]
    for n in (1, 5, 16):
        check_nv12(mode, ui, 130, 74, [("clip", n), ("clip", n), ("frame",), ("frame",)], launches=True)


@pytest.mark.parametrize("mname", list(MODES))
def test_nv12_and_bgr_calls_interleave_on_one_handle(mname):
    mode, ui = MODES[mname]
    check_nv12(mode, ui, 130, 74, [("frame",), ("bgr",), ("frame",), ("clip", 3), ("bgr",), ("frame",)])


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_lanes_restart_and_hold(mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("frame",), ("restart", 2), ("hold", 1, 1), ("frame",), ("frame",), ("hold", 1, 0), ("frame",),
             ("restart", 0), ("hold", 3, 1), ("clip", 4), ("hold", 3, 0), ("clip", 3)]
    check_nv12(mode, ui, 130, 74, steps, lanes=4, launches=True)


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("layout", ["odd_pitch", "padded", "uv_offset"])
def test_padded_pitches_and_plane_offsets(mname, layout):
    """odd pitch (byte path), 64-byte pitch with spare rows between lanes, and the Cb,Cr plane 30 rows below the luma"""
    mode, ui = MODES[mname]
    w, h = 130, 74
    lay = {"odd_pitch": Layout(w, h, pitch=133), "padded": Layout(w, h, pitch=192, rows=h * 3 // 2 + 5),
           "uv_offset": Layout(w, h, pitch=136, uv_row=h + 30)}[layout]
    check_nv12(mode, ui, w, h, [("frame",), ("frame",), ("clip", 3), ("frame",)], lanes=2, layout=lay)


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("kind", ["blocks", "checker", "shadows", "highlights", "corners", "noise"])
def test_full_range_content(mname, kind):
    mode, ui = MODES[mname]
    check_nv12(mode, ui, 242, 136, [("frame",), ("frame",), ("clip", 4), ("frame",)], lanes=2, kind=kind)


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
@pytest.mark.parametrize("mname", list(MODES))
def test_1080p_decoder_surface(mname):
    """1920 x 1080 with the Cb,Cr plane at row 1088, as a decoder surface puts it"""
    mode, ui = MODES[mname]
    lay = Layout(1920, 1080, pitch=2048, uv_row=1088)
    check_nv12(mode, ui, 1920, 1080, [("frame",), ("frame",), ("clip", 5), ("frame",)], lanes=2, layout=lay)


# ---- the pipelined host path ----------------------------------------------------------------------------------------

def _pinned(lib, shape, keep):
    p = lib.mc_host_alloc(int(np.prod(shape)))
    keep.append(p)
    return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=shape)


def check_submit_nv12(mname, pinned, layout, w, h):
    """Three frames in flight, restarts and holds taken at submit: mc_submit_nv12 / mc_collect give the device calls'
    planes and flags; both planes of lanes that did not produce keep the sentinel."""
    mode, ui = MODES[mname]
    cfg, _ = make_cfgs(mode, *ui)
    lanes, n, depth = 4, 9, 3
    lay = Layout(w, h) if layout == "packed" else Layout(w, h, pitch=w + 6, uv_row=h + 6)
    events = {1: [("hold", 3, 1)], 2: [("restart", 0)], 4: [("hold", 3, 0), ("restart", 2)],
              5: [("restart", 1), ("hold", 2, 1)], 7: [("hold", 2, 0)]}

    def apply(p, t):
        for e in events.get(t, []):
            p.hold_lane(e[1], e[2]) if e[0] == "hold" else p.restart_lane(e[1])

    frames = [lay.pack(np.stack([to_nv12(f) for f in source(t, 1, lanes, w, h, None)[0]])) for t in range(n)]
    ref_dev, sub = proc(lanes), proc(lanes)
    ref = []
    for t in range(n):
        apply(ref_dev, t)
        d_in, d_out = Dev(frames[t]), Dev(np.full_like(frames[t], SENTINEL))
        prod = ref_dev.process_nv12_device(lay.planes(d_in.ptr), w, h, cfg, lay.planes(d_out.ptr))
        ref_dev.sync()
        ref.append((prod, ref_dev.lane_produced(), d_out.numpy()))
    lib, keep = capi.lib(), []
    try:
        if pinned:
            ins = [_pinned(lib, frames[0].shape, keep) for _ in range(n)]
            outs = [_pinned(lib, frames[0].shape, keep) for _ in range(n)]
            for t in range(n):
                ins[t][...] = frames[t]
        else:
            ins, outs = frames, [np.empty_like(frames[0]) for _ in range(n)]
        for o in outs:
            o[...] = SENTINEL
        got, done = [], 0
        for t in range(n):
            if t - done >= depth:
                got.append((sub.collect(), sub.lane_produced()))
                done += 1
            apply(sub, t)
            sub.submit_nv12(lay.planes(ins[t].ctypes.data), w, h, cfg, lay.planes(outs[t].ctypes.data))
        while done < n:
            got.append((sub.collect(), sub.lane_produced()))
            done += 1
        for t in range(n):
            assert got[t][0] == ref[t][0], t
            assert np.array_equal(got[t][1], ref[t][1]), t
            assert np.array_equal(outs[t], ref[t][2]), t
        assert not all(r[1].all() for r in ref)   # some frames leave lanes untouched
    finally:
        sub.close()
        for p in keep:
            lib.mc_host_free(p)


@pytest.mark.parametrize("mname", ["laplace", "phase"])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("layout", ["packed", "uv_offset"])
def test_submit_nv12_equals_device_calls(mname, pinned, layout):
    check_submit_nv12(mname, pinned, layout, 130, 74)


def test_bad_arguments_leave_state_untouched():
    """odd or too small sizes, null planes, pitch < width, overlapping lanes: MC_ERR_INVALID, and the next valid call
    equals that of a handle that never saw the bad ones"""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    w, h, lanes = 130, 74, 2
    lay = Layout(w, h)
    a, b = proc(lanes), proc(lanes)
    lib = capi.lib()
    prm = _to_mc(cfg)
    x = [lay.pack(np.stack([to_nv12(f) for f in source(t, 1, lanes, w, h, None)[0]])) for t in range(3)]
    d_in, d_out = Dev(x[0]), Dev(np.zeros_like(x[0]))
    for p in (a, b):
        p.process_nv12_device(lay.planes(d_in.ptr), w, h, cfg, lay.planes(d_out.ptr))
    good_in, good_out = lay.planes(d_in.ptr), lay.planes(d_out.ptr)
    bad = [(w + 1, h, good_in, good_out), (w, h - 1, good_in, good_out), (0, 0, good_in, good_out),
           (w, h, capi.McNv12(None, good_in.uv, lay.pitch, lay.lane_stride), good_out),
           (w, h, good_in, capi.McNv12(good_out.y, None, lay.pitch, lay.lane_stride)),
           (w, h, capi.McNv12(good_in.y, good_in.uv, w - 2, lay.lane_stride), good_out),
           (w, h, good_in, capi.McNv12(good_out.y, good_out.uv, lay.pitch, lay.pitch * h - 1))]
    produced, flags = C.c_int(7), np.zeros((2, lanes), np.uint8)
    for ww, hh, i, o in bad:
        assert lib.mc_process_nv12_device(a._h, C.byref(i), ww, hh, C.byref(prm), C.byref(o), C.byref(produced)) == capi.MC_ERR_INVALID
        assert produced.value == 0
        assert lib.mc_process_clip_nv12_device(a._h, C.byref(i), 2, ww, hh, C.byref(prm), C.byref(o),
                                               flags.ctypes.data_as(C.POINTER(C.c_uint8))) == capi.MC_ERR_INVALID
        assert lib.mc_submit_nv12(a._h, C.byref(i), ww, hh, C.byref(prm), C.byref(o)) == capi.MC_ERR_INVALID
    for bad_frames in (0, capi.MC_MAX_LANES):
        assert lib.mc_process_clip_nv12_device(a._h, C.byref(good_in), bad_frames, w, h, C.byref(prm), C.byref(good_out),
                                               flags.ctypes.data_as(C.POINTER(C.c_uint8))) == capi.MC_ERR_INVALID
    for t in (1, 2):
        outs = []
        for p in (a, b):
            di, do = Dev(x[t]), Dev(np.full_like(x[t], SENTINEL))
            assert p.process_nv12_device(lay.planes(di.ptr), w, h, cfg, lay.planes(do.ptr))
            p.sync()
            outs.append(do.numpy())
        assert np.array_equal(outs[0], outs[1]), t
    assert_states_equal(a, b, O.MODE_LAPLACE)


# ---- the two kernels alone, on every input --------------------------------------------------------------------------

def yuv_sets(w):
    """-> 64 packed NV12 frames [64][3h/2][w] that hold every (Y, Cb, Cr) triple: every (Cb, Cr) pair is one 2x2 block
    (repeated to fill the last block row), and frame f gives its block's four pixels the luma values 4f .. 4f+3."""
    nb = w // 2
    bh = -(-65536 // nb)
    pair = np.arange(bh * nb) % 65536
    uv = np.stack([pair >> 8, pair & 255], -1).astype(np.uint8).reshape(bh, w)
    out = []
    for f in range(64):
        y = np.broadcast_to(np.arange(4 * f, 4 * f + 4, dtype=np.uint8).reshape(1, 2, 1, 2), (bh, 2, nb, 2)).reshape(2 * bh, w)
        out.append(np.concatenate([y, uv]))
    return np.stack(out)


def bgr_sets(w, lanes, seed=3):
    """-> BGR [lanes][h][w][3] in which every 24-bit colour is the top-left pixel of a 2x2 block (repeated to fill the last
    block row); the other three pixels of each block are random"""
    nb = w // 2
    bh = -(-(1 << 24) // (nb * lanes))
    idx = np.arange(lanes * bh * nb, dtype=np.uint32) % (1 << 24)
    tl = np.stack([idx & 255, (idx >> 8) & 255, idx >> 16], -1).astype(np.uint8).reshape(lanes, bh, nb, 3)
    img = np.random.default_rng(seed).integers(0, 256, (lanes, 2 * bh, w, 3), dtype=np.uint8)
    img[:, ::2, ::2] = tl
    return img


def _debug(name):
    fn = getattr(capi.lib(), name)
    fn.restype = C.c_int
    return fn


@pytest.mark.skipif(EMU, reason="every colour is too slow for the CPU emulation")
@pytest.mark.parametrize("w,pitch,uv_row_pad,bgr_pad", [(4096, 4096, 0, 0), (4090, 4091, 3, 1), (4096, 4104, 1024, 8)])
def test_nv12_to_bgr_kernel_on_every_yuv(w, pitch, uv_row_pad, bgr_pad):
    """aligned 4096-wide frames; width = 2 mod 8 with an odd pitch and unaligned BGR rows (the byte paths and the tails);
    a padded pitch with the Cb,Cr plane 1024 rows further down.  64 frames as 64 lanes of one launch."""
    nv = yuv_sets(w)
    h = nv.shape[1] * 2 // 3
    lay = Layout(w, h, pitch=pitch, uv_row=h + uv_row_pad)
    step = 3 * w + bgr_pad
    d_in, d_bgr = Dev(lay.pack(nv)), Dev(np.zeros((len(nv), h, step), np.uint8))
    planes = lay.planes(d_in.ptr)
    assert _debug("mc_debug_nv12_to_bgr")(C.byref(planes), w, h, len(nv), C.c_void_p(d_bgr.ptr), C.c_size_t(step)) == 0
    got = d_bgr.numpy()
    for f in range(len(nv)):
        assert np.array_equal(got[f, :, :3 * w].reshape(h, w, 3), to_bgr(nv[f])), f
        assert (got[f, :, 3 * w:] == 0).all()


@pytest.mark.skipif(EMU, reason="every colour is too slow for the CPU emulation")
@pytest.mark.parametrize("w,pitch,uv_row_pad,bgr_pad", [(4096, 4096, 0, 0), (4090, 4091, 3, 1), (4096, 4104, 1024, 8)])
def test_bgr_to_nv12_kernel_on_every_colour(w, pitch, uv_row_pad, bgr_pad):
    """every colour as a block's top-left pixel, over 4 lanes; then the same with lanes 1 and 3 flagged off: their
    planes are not written"""
    lanes = 4
    img = bgr_sets(w, lanes)
    h = img.shape[1]
    step = 3 * w + bgr_pad
    buf = np.zeros((lanes, h, step), np.uint8)
    buf[:, :, :3 * w] = img.reshape(lanes, h, 3 * w)
    lay = Layout(w, h, pitch=pitch, uv_row=h + uv_row_pad)
    d_bgr = Dev(buf)
    want = lay.pack(np.stack([to_nv12(f) for f in img]))
    fn = _debug("mc_debug_bgr_to_nv12")
    for flags in (None, np.array([1, 0, 1, 0], np.uint8)):
        d_out = Dev(np.full_like(want, SENTINEL))
        d_flags = Dev(flags) if flags is not None else None
        assert fn(C.c_void_p(d_bgr.ptr), C.c_size_t(step), w, h, lanes, C.c_void_p(d_flags.ptr if d_flags else None),
                  C.byref(lay.planes(d_out.ptr))) == 0
        got = d_out.numpy()
        for k in range(lanes):
            if flags is None or flags[k]:
                assert np.array_equal(got[k], want[k]), k
            else:
                assert (got[k] == SENTINEL).all(), k
