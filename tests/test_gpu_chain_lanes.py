"""The processing chain on device frames, for every lane and in clips (mc_chain_process_device), and straight from NV12
planes (mc_chain_process_nv12_device).

The front kernel alone (mode None) is checked against cv2 bit for bit; a multi-lane chain against one 1-lane
mc_chain_process handle per lane (processed frame, original tap, info, flags, state); clips against frame calls; the NV12
chain against the BGR chain on cv2's conversion; one 4K -> 1080p case against the oracle; and the error cases, which
must return before any launch with every buffer and the state unchanged."""
import ctypes as C
import os

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs, u8_diff
from test_gpu_lanes import LAPLACE_UI, PHASE_UI, COLOR_UI, SENTINEL, lane_frame, state_names
from test_gpu_nv12 import Dev, Layout, to_bgr, to_nv12

EMU = os.environ.get("MC_EMU") == "1"
MODES = {"laplace": (O.MODE_LAPLACE, LAPLACE_UI), "phase": (O.MODE_PHASE, PHASE_UI), "color": (O.MODE_COLOR, COLOR_UI)}


# ---- configurations, sources and one device call ---------------------------------------------------------------------

def chain_cfg(mode, ui, down=1, roi=None, gray=False):
    cfg, _ = make_cfgs(mode, *ui)
    cfg.grayscale = gray
    cfg.preprocess = L.PreprocessParams(down, roi is not None, *(roi if roi else (0.0, 0.0, 1.0, 1.0)))
    return cfg


def none_cfg(down=1, roi=None, gray=False):
    return chain_cfg(O.MODE_NONE, LAPLACE_UI, down, roi, gray)


def full_range(v, w, h, c, seed=0):
    """v frames [v][h][w](c) of uniform random bytes"""
    shape = (v, h, w) + ((c,) if c == 3 else ())
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def as_nv12(bgr):
    """BGR frames -> (packed NV12 frames, their cv2 conversion back to BGR: what the NV12 chain must equal)"""
    nv = np.stack([to_nv12(f) for f in bgr])
    return nv, np.stack([to_bgr(f) for f in nv])


def out_geom(ch, cfg, w, h, c):
    """-> (rows, row bytes) of d_out and of d_original for a w x h x c source (the input's where a stage is an identity)"""
    g = ch.geometry(cfg, w, h, c)
    out = (h, w * c) if g.cur_is_input else (g.out_h, g.out_w * g.out_channels)
    orig = (h, w * c) if g.orig_is_input else (g.orig_h, g.orig_w * g.orig_channels)
    return out, orig


def device_call(ch, cfg, src, frames, w, h, c, nv12=None, in_pad=0, out_pad=0, orig_pad=0, want_orig=True):
    """One chain call on V = frames * lanes source frames (src [V][h][w](c); with nv12 = a Layout, packed NV12 frames) into
    sentinel-filled buffers -> (flags u8 [frames, lanes], info, out [V][rows][step], orig [V][rows][step] or None)"""
    (oh, orow), (gh, grow) = out_geom(ch, cfg, w, h, c)
    v = len(src)
    out_step, orig_step = orow + out_pad, grow + orig_pad
    d_out = Dev(np.full((v, oh, out_step), SENTINEL, np.uint8))
    d_orig = Dev(np.full((v, gh, orig_step), SENTINEL, np.uint8)) if want_orig else None
    if nv12 is not None:
        d_in = Dev(nv12.pack(src, fill=0x3C))
        flags, info = ch.process_nv12_device(nv12.planes(d_in.ptr), frames, w, h, cfg, d_out.ptr, out_step,
                                             d_orig.ptr if d_orig else 0, orig_step)
    else:
        in_step = w * c + in_pad
        buf = np.full((v, h, in_step), 0x3C, np.uint8)
        buf[:, :, :w * c] = src.reshape(v, h, w * c)
        d_in = Dev(buf)
        flags, info = ch.process_device(d_in.ptr, frames, w, h, c, in_step, cfg, d_out.ptr, out_step,
                                        d_orig.ptr if d_orig else 0, orig_step)
    ch.magnifier.sync()
    return flags.astype(np.uint8), info, d_out.numpy(), d_orig.numpy() if d_orig else None


def expected(shape, row, images):
    """sentinel-filled [V][rows][step] with images[v] (None: untouched) in its first `row` bytes"""
    want = np.full(shape, SENTINEL, np.uint8)
    for v, im in enumerate(images):
        if im is not None:
            want[v, :, :row] = im.reshape(shape[1], row)
    return want


def info_tuple(i):
    return (i.cur_is_input, i.out_w, i.out_h, i.out_channels, i.orig_is_input, i.orig_w, i.orig_h, i.orig_channels, i.magnified)


# ---- the chain against one 1-lane mc_chain_process handle per lane ----------------------------------------------------

def check_chain(mode, ui, w, h, c, steps, lanes=4, nv12=None, options=(), launches=False):
    """A `lanes`-lane chain handle takes device calls; lane k's reference is a 1-lane ProcessingChainB200 fed lane k's frames
    one run_chain_once at a time (not fed while held).  steps: ("frame",) / ("clip", n) device calls; ("restart", k) /
    ("hold", k, on) on the multi-lane handle and the reference of lane k; ("cfg", kwargs) new chain settings
    (down / roi / gray) from here on.  nv12: a Layout; the sources are then NV12 frames and the references take cv2's
    conversion.  Each call's d_out and d_original (sentinel-filled, padding included), flags and info must be the
    references'; at the end every lane's state planes are its reference's.  launches: every call launches chain_front
    once when a front stage is on, none otherwise (and no nv12_to_bgr with a front stage)."""
    settings = {}
    cfg = chain_cfg(mode, ui)
    opts = tuple(options) + ((("profile_kernels", 1),) if launches else ())
    multi = L.ProcessingChainB200(0, lanes=lanes)
    refs = [L.ProcessingChainB200(0) for _ in range(lanes)]
    for k, val in opts:
        multi.magnifier.set_option(k, val)
    held = [False] * lanes
    t = 0
    for step in steps:
        if step[0] == "restart":
            multi.magnifier.restart_lane(step[1])
            refs[step[1]].reset()
            continue
        if step[0] == "hold":
            multi.magnifier.hold_lane(step[1], step[2])
            held[step[1]] = bool(step[2])
            continue
        if step[0] == "cfg":
            settings = step[1]
            cfg = chain_cfg(mode, ui, **settings)
            continue
        n = step[1] if step[0] == "clip" else 1
        bgr = np.stack([lane_frame(s, k, w, h, c) for s in range(t, t + n) for k in range(lanes)])
        t += n
        src, ref_in = (bgr, bgr) if nv12 is None else as_nv12(bgr)
        if launches:
            multi.magnifier.profile_read()
        flags, info, out, orig = device_call(multi, cfg, src, n, w, h, c, nv12=nv12)
        outs, origs, want_flags, magnified = [], [], np.zeros((n, lanes), np.uint8), 0
        for v in range(n * lanes):
            k = v % lanes
            if held[k]:
                outs.append(None)
                origs.append(None)
                continue
            fr = L.Frame(image=ref_in[v])
            cur, original = refs[k].run_chain_once(fr, cfg)
            ref_prod = refs[k].magnifier.lane_produced()[0]
            want_flags[v // lanes, k] = ref_prod
            magnified |= int(ref_prod)
            outs.append(None if cur is fr else cur.image)
            origs.append(None if original is fr else original.image)
        geo = L.ProcessingChainB200.geometry(cfg, w, h, c)
        assert np.array_equal(flags, want_flags), (step, flags, want_flags)
        assert info_tuple(info) == info_tuple(geo)[:-1] + (magnified,), (step, info_tuple(info))
        assert np.array_equal(multi.magnifier.lane_produced(), want_flags[-1].astype(bool))
        (_, orow), (_, grow) = out_geom(multi, cfg, w, h, c)
        assert np.array_equal(out, expected(out.shape, orow, outs)), step
        assert np.array_equal(orig, expected(orig.shape, grow, origs)), step
        if launches:
            comp = {k: v[0] for k, v in multi.magnifier.profile_read().items()}
            front = not (geo.cur_is_input and geo.orig_is_input)
            assert comp.get(("chain_front", 0), 0) == (1 if front else 0), (step, comp)
            if front:
                assert ("nv12_to_bgr", 0) not in comp
    if mode != O.MODE_NONE:
        names = state_names(refs[0].magnifier, mode)
        assert names == state_names(multi.magnifier, mode)
        for n_, l in names:
            got = multi.magnifier.get_state(n_, l)
            for k in range(lanes):
                assert np.array_equal(got[k], refs[k].magnifier.get_state(n_, l)[0]), (n_, l, k)
    return multi


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu

FRONT_CASES = [
    # (w, h, down, roi, gray, in_pad, out_pad, lanes, frames)
    *[(66, 50, d, None, False, 0, 0, 1, 1) for d in range(1, 9)],
    (642, 478, 3, (0.1, 0.2, 0.77, 0.61), True, 0, 0, 1, 1),      # fractional INTER_AREA scale
    (640, 480, 4, None, True, 7, 3, 1, 1),                         # integer scale, padded steps
    (200, 150, 2, (0.997, 0.995, 0.5, 0.5), False, 0, 0, 1, 1),    # ROI at the last column / row: 1 x 1
    (200, 150, 3, (0.5, 0.0, 0.9, 1.5), True, 1, 1, 1, 1),         # ROI larger than what is left of the frame
    (206, 154, 2, None, False, 0, 5, 1, 1),                        # odd output sizes: 103 x 77
    (202, 152, 1, (0.015, 0.0, 0.5, 1.0), True, 0, 0, 1, 1),      # crop at an odd column, gray
    (130, 74, 1, None, True, 0, 0, 1, 1),                          # gray alone
    (130, 74, 5, (0.1, 0.1, 0.8, 0.8), True, 0, 0, 3, 4),          # several virtual lanes
]


@pytest.mark.parametrize("src", ["bgr", "gray", "nv12"])
@pytest.mark.parametrize("w,h,down,roi,gray,in_pad,out_pad,lanes,frames", FRONT_CASES)
def test_front_matches_cv2(src, w, h, down, roi, gray, in_pad, out_pad, lanes, frames):
    """Mode None: d_out is the front's output and d_original the preprocessed frame, each bit for bit cv2's (the oracle's
    preprocess() and grayscale() call cv2.resize(INTER_AREA) and cv2.cvtColor); bytes outside the rows are untouched."""
    c = 1 if src == "gray" else 3
    cfg = none_cfg(down, roi, gray)
    ocfg = O.ProcessorConfig(grayscale=gray, preprocess=O.PreprocessParams(down, roi is not None, *(roi or (0.0, 0.0, 1.0, 1.0))))
    ch = L.ProcessingChainB200(0, lanes=lanes)
    v = lanes * frames
    data = full_range(v, w, h, c, seed=w + down)
    nv = None
    if src == "nv12":
        data, bgr = as_nv12(data)
        nv = Layout(w, h, pitch=w + 3 if in_pad else w)
    else:
        bgr = data
    flags, info, out, orig = device_call(ch, cfg, data, frames, w, h, c, nv12=nv, in_pad=in_pad, out_pad=out_pad, orig_pad=out_pad)
    assert not flags.any() and not info.magnified
    pre = [O.preprocess(f, ocfg) for f in bgr]
    cur = [O.grayscale(p[1], ocfg) for p in pre]
    front = pre[0][0] or cur[0][0]
    assert info.orig_is_input == (not pre[0][0]) and info.cur_is_input == (not front)
    if pre[0][0]:
        assert (info.orig_h, info.orig_w, info.orig_channels) == (pre[0][1].shape[0], pre[0][1].shape[1], c)
    (_, orow), (_, grow) = out_geom(ch, cfg, w, h, c)
    assert np.array_equal(out, expected(out.shape, orow, [g[1] if front else None for g in cur]))
    assert np.array_equal(orig, expected(orig.shape, grow, [p[1] if p[0] else None for p in pre]))


@pytest.mark.skipif(EMU, reason="4K frames are too slow for the CPU emulation")
@pytest.mark.parametrize("gray", [False, True])
def test_front_4k_nv12_decoder_surface_to_1080p(gray):
    """3840 x 2160 NV12 with a padded pitch and the Cb,Cr plane at row 2176 (a decoder surface), 2 lanes, downscale 2"""
    w, h = 3840, 2160
    cfg = none_cfg(2, None, gray)
    ocfg = O.ProcessorConfig(grayscale=gray, preprocess=O.PreprocessParams(2, False, 0.0, 0.0, 1.0, 1.0))
    ch = L.ProcessingChainB200(0, lanes=2)
    nv, bgr = as_nv12(full_range(2, w, h, 3, seed=4))
    flags, info, out, orig = device_call(ch, cfg, nv, 1, w, h, 3, nv12=Layout(w, h, pitch=4096, uv_row=2176))
    assert (info.out_w, info.out_h) == (1920, 1080)
    for k in range(2):
        pre = O.preprocess(bgr[k], ocfg)[1]
        assert np.array_equal(orig[k].reshape(pre.shape), pre), k
        assert np.array_equal(out[k].reshape(-1), O.grayscale(pre, ocfg)[1].reshape(-1)), k


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_lanes_equal_single_chains_with_restart_hold_and_roi_move(mname):
    mode, ui = MODES[mname]
    steps = [("cfg", dict(down=3, roi=(0.1, 0.2, 0.77, 0.61), gray=False)), ("frame",), ("frame",), ("restart", 2),
             ("hold", 1, 1), ("frame",), ("clip", 3), ("hold", 1, 0), ("frame",),
             ("cfg", dict(down=3, roi=(0.15, 0.2, 0.77, 0.61), gray=False)),   # the ROI moves: every lane restarts
             ("frame",), ("restart", 0), ("hold", 3, 1), ("clip", 2), ("hold", 3, 0), ("frame",)]
    check_chain(mode, ui, 241, 163, 3, steps, lanes=4, launches=True)


def test_lanes_equal_single_chains_color():
    mode, ui = MODES["color"]
    steps = [("cfg", dict(down=2, roi=(0.1, 0.1, 0.8, 0.8), gray=True)), ("frame",), ("clip", 3), ("frame",),
             ("cfg", dict(down=2, roi=(0.12, 0.1, 0.8, 0.8), gray=True)), ("clip", 4), ("frame",)]
    check_chain(mode, ui, 240, 180, 3, steps, lanes=4, launches=True)


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("front", [dict(down=2, gray=True), dict(down=1)], ids=["front", "no_front"])
def test_clips_equal_frame_calls(mname, front):
    """T = 1, 5, 16 from a fresh handle (Phase's first frame, Color's warm-up inside the clip): frames that did not produce
    carry the front's output when a front stage ran and leave d_out untouched otherwise"""
    mode, ui = MODES[mname]
    for n in (1, 5, 16):
        check_chain(mode, ui, 130, 74, 3, [("cfg", front), ("clip", n), ("clip", n), ("frame",)], lanes=2, launches=True)


@pytest.mark.parametrize("mname", list(MODES))
@pytest.mark.parametrize("settings", [dict(down=2, roi=(0.05, 0.1, 0.9, 0.85), gray=False), dict(down=3, gray=True),
                                      dict(down=1, gray=True), dict(down=1)], ids=["crop_down", "down_gray", "gray", "none"])
def test_nv12_chain_equals_bgr_chain_on_cv2_conversion(mname, settings):
    """The references take cv2's COLOR_YUV2BGR_NV12 of each NV12 frame: frames, clips and a hold, with an odd pitch and the
    Cb,Cr plane 6 rows below the luma; "gray" is gray magnification of an NV12 source"""
    mode, ui = MODES[mname]
    lay = Layout(130, 74, pitch=133, uv_row=80)
    hold = [] if mname == "color" else [("hold", 1, 1), ("frame",), ("hold", 1, 0)]
    steps = [("cfg", settings), ("frame",), ("clip", 3), *hold, ("clip", 2), ("frame",)]
    check_chain(mode, ui, 130, 74, 3, steps, lanes=2, nv12=lay, launches=True)


@pytest.mark.skipif(EMU, reason="4K frames are too slow for the CPU emulation")
def test_4k_to_1080p_against_the_oracle():
    """4K source, downscale 2, 1080p Laplace on 2 lanes: d_original bit-exact, d_out within the chain's tolerance"""
    w, h, lanes = 3840, 2160, 2
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 20, 6)
    cfg.preprocess, ocfg.preprocess = L.PreprocessParams(2), O.PreprocessParams(2)
    ch = L.ProcessingChainB200(0, lanes=lanes)
    omags = [O.MagnificationProcessor() for _ in range(lanes)]
    for t in range(2):
        src = np.stack([lane_frame(t, k, w, h, 3) for k in range(lanes)])
        flags, info, out, orig = device_call(ch, cfg, src, 1, w, h, 3)
        assert flags.all() and info.magnified and (info.out_w, info.out_h) == (1920, 1080)
        for k in range(lanes):
            ocur, oorig, _, _ = O.run_chain_once(omags[k], src[k], ocfg)
            assert np.array_equal(orig[k].reshape(oorig.shape), oorig), (t, k)
            assert int(u8_diff(out[k].reshape(ocur.shape), ocur).max()) <= 1, (t, k)


def _raw(ch, cfg, d_in, frames, w, h, c, in_step, d_out, out_step, d_orig, orig_step, flags, nv12=None):
    lib, m, p, info = capi.lib(), ch.magnifier, _to_mc(cfg), capi.McChainInfo()
    u8 = flags.ctypes.data_as(C.POINTER(C.c_uint8)) if flags is not None else None
    if nv12 is not None:
        return lib.mc_chain_process_nv12_device(m._h, C.byref(nv12), frames, w, h, C.byref(p), int(cfg.grayscale), d_out,
                                                out_step, d_orig, orig_step, u8, C.byref(info))
    return lib.mc_chain_process_device(m._h, d_in, frames, w, h, c, in_step, C.byref(p), int(cfg.grayscale), d_out, out_step,
                                       d_orig, orig_step, u8, C.byref(info))


def test_errors_return_before_any_launch():
    """Each bad call returns its status with the launch count, both output buffers and every state plane unchanged; Color's
    refusal with a held lane is MC_ERR_UNSUPPORTED, and pipelined frames in flight are refused"""
    w, h, c, lanes = 130, 74, 3, 2
    src = np.stack([lane_frame(0, k, w, h, c) for k in range(lanes)])
    nv, _ = as_nv12(src)
    lay = Layout(w, h)
    d_in, d_nv = Dev(np.ascontiguousarray(src)), Dev(lay.pack(nv))
    good = lay.planes(d_nv.ptr)

    def setup(cfg):
        ch = L.ProcessingChainB200(0, lanes=lanes)
        device_call(ch, cfg, src, 1, w, h, c)                 # state to keep
        (oh, orow), (gh, grow) = out_geom(ch, cfg, w, h, c)
        bufs = Dev(np.full((4 * lanes, oh, orow), SENTINEL, np.uint8)), Dev(np.full((4 * lanes, gh, grow), SENTINEL, np.uint8))
        args = dict(d_in=d_in.ptr, frames=1, w=w, h=h, c=c, in_step=w * c, d_out=bufs[0].ptr, out_step=orow, d_orig=bufs[1].ptr,
                    orig_step=grow, flags=np.zeros((4, lanes), np.uint8))
        return ch, bufs, args

    def unchanged(ch, bufs, mode, before, n0):
        m = ch.magnifier
        m.sync()
        assert m.launch_count == n0
        assert all((b.numpy() == SENTINEL).all() for b in bufs)
        names = state_names(m, mode)
        assert all(np.array_equal(m.get_state(n, l), a) for (n, l), a in zip(names, before))

    cfg = chain_cfg(O.MODE_LAPLACE, LAPLACE_UI, down=2, roi=(0.1, 0.1, 0.8, 0.8), gray=True)
    ch, bufs, args = setup(cfg)
    m = ch.magnifier
    before, n0 = [m.get_state(n, l) for n, l in state_names(m, O.MODE_LAPLACE)], m.launch_count
    bad = [dict(in_step=w * c - 1), dict(out_step=args["out_step"] - 1), dict(orig_step=args["orig_step"] - 1), dict(d_out=None),
           dict(frames=0), dict(frames=capi.MC_MAX_LANES), dict(flags=None), dict(c=2),
           dict(nv12=capi.McNv12(good.y, good.uv, w - 1, good.lane_stride)), dict(nv12=good, w=w - 1),
           dict(nv12=capi.McNv12(good.y, None, good.pitch, good.lane_stride)),
           dict(nv12=capi.McNv12(good.y, good.uv, good.pitch, good.pitch * h - 1))]
    for b in bad:
        assert _raw(ch, cfg, **{**args, **b}) == capi.MC_ERR_INVALID, b
    unchanged(ch, bufs, O.MODE_LAPLACE, before, n0)

    color = chain_cfg(O.MODE_COLOR, COLOR_UI, down=2, gray=True)
    ch, bufs, args = setup(color)
    ch.magnifier.hold_lane(1, True)
    n0 = ch.magnifier.launch_count
    for nv12 in (None, good):
        assert _raw(ch, color, **args, nv12=nv12) == capi.MC_ERR_UNSUPPORTED
    unchanged(ch, bufs, O.MODE_COLOR, [], n0)

    ch, bufs, args = setup(cfg)
    out = np.empty_like(src)
    ch.magnifier.submit(src.ctypes.data, w, h, c, w * c, cfg, out.ctypes.data, w * c)
    n0 = ch.magnifier.launch_count
    assert _raw(ch, cfg, **args) == capi.MC_ERR_INVALID
    assert ch.magnifier.launch_count == n0
    ch.magnifier.collect()


def test_launches_and_profile_name():
    """One chain_front launch per call with a front stage; mode None without front stages launches nothing at all"""
    w, h, c, lanes = 130, 74, 3, 2
    src = np.stack([lane_frame(0, k, w, h, c) for k in range(lanes)])
    ch = L.ProcessingChainB200(0, lanes=lanes)
    ch.magnifier.set_option("profile_kernels", 1)
    n0 = ch.magnifier.launch_count
    device_call(ch, none_cfg(), src, 1, w, h, c)
    assert ch.magnifier.launch_count == n0 and not ch.magnifier.profile_read()
    for cfg in (none_cfg(2), none_cfg(1, None, True), chain_cfg(O.MODE_LAPLACE, LAPLACE_UI, 3, (0.1, 0.1, 0.7, 0.7), True)):
        device_call(ch, cfg, src, 1, w, h, c)
        assert ch.magnifier.profile_read()[("chain_front", 0)][0] == 1
