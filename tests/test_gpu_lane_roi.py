"""Per-lane regions of interest (mc_set_lane_roi): lane k of a multi-lane chain handle, with the call's params where its
override replaces the four ROI fields, must equal, bit for bit, a 1-lane ProcessingChainB200 fed lane k's frames with
those params: processed frames, original taps, canvases, info, produced flags, mc_lane_produced and the temporal state
afterwards (mc_save_lane blobs; Color through its window taps, since a Color blob also carries unfilled ring slots).  A
lane whose ROI moves restarts alone, as its twin's structural reset does; the other lanes run on untouched."""
import ctypes as C
import dataclasses

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.labels import export_labels
from oracle import livim_oracle as O
from test_gpu_chain_lanes import MODES, chain_cfg, info_tuple
from test_gpu_lanes import SENTINEL, lane_frame, state_names
from test_gpu_nv12 import EMU, Dev, to_nv12
from test_gpu_rgb import from_bgr as rgb_of
from test_gpu_yuv422 import from_bgr as yuyv_of

pytestmark = pytest.mark.gpu

SOURCES = ("bgr", "gray", "nv12", "yuyv", "uyvy", "i420", "yv12", "rgb", "rgba", "bgra", "rgb_planar")
RGB_LAYOUT = {"rgb": capi.MC_RGB_RGB, "rgba": capi.MC_RGB_RGBA, "bgra": capi.MC_RGB_BGRA, "rgb_planar": capi.MC_RGB_PLANAR}


# ---- sources ---------------------------------------------------------------------------------------------------------
def pack(kind, bgr):
    """BGR frames [V][h][w][3] -> the source frames of `kind`, one dense frame per virtual lane"""
    if kind == "bgr":
        return np.ascontiguousarray(bgr)
    if kind == "gray":
        return np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in bgr])
    if kind == "nv12":
        return np.stack([to_nv12(f) for f in bgr])
    if kind in ("yuyv", "uyvy"):
        return np.stack([yuyv_of(f, capi.MC_YUV422_YUYV if kind == "yuyv" else capi.MC_YUV422_UYVY) for f in bgr])
    if kind in ("i420", "yv12"):
        return np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in bgr])
    return np.stack([rgb_of(f, RGB_LAYOUT[kind]) for f in bgr])


def call(ch, kind, cfg, frames, w, h, dev, d_out, out_step, d_orig, orig_step):
    """One device chain call of `kind` on the packed frames in `dev`, complete when it returns -> (flags bool [frames,
    lanes], info)"""
    r = dispatch(ch, kind, cfg, frames, w, h, dev, d_out, out_step, d_orig, orig_step)
    ch.magnifier.sync()   # the handle's stream does not order with the one the buffers are read back on
    return r


def dispatch(ch, kind, cfg, frames, w, h, dev, d_out, out_step, d_orig, orig_step):
    p, n, lane = dev.ptr, w * h, dev.lane_bytes
    if kind in ("bgr", "gray"):
        c = 3 if kind == "bgr" else 1
        return ch.process_device(p, frames, w, h, c, w * c, cfg, d_out, out_step, d_orig, orig_step)
    if kind == "nv12":
        return ch.process_nv12_device(capi.McNv12(p, p + n, w, lane), frames, w, h, cfg, d_out, out_step, d_orig, orig_step)
    if kind in ("yuyv", "uyvy"):
        order = capi.MC_YUV422_YUYV if kind == "yuyv" else capi.MC_YUV422_UYVY
        return ch.process_yuv422_device(capi.McYuv422(p, 2 * w, lane, order), frames, w, h, cfg, d_out, out_step, d_orig, orig_step)
    if kind in ("i420", "yv12"):
        u, v = p + n, p + n + n // 4
        if kind == "yv12":
            u, v = v, u
        return ch.process_yuv420p_device(capi.McYuv420p(p, u, v, w, w // 2, lane), frames, w, h, cfg, d_out, out_step, d_orig,
                                         orig_step)
    layout = RGB_LAYOUT[kind]
    if layout == capi.MC_RGB_PLANAR:
        s = capi.McRgb(p, p + n, p + 2 * n, w, lane, layout)
    else:
        bpp = 3 if layout == capi.MC_RGB_RGB else 4
        s = capi.McRgb(p, None, None, w * bpp, lane, layout)
    return ch.process_rgb_device(s, frames, w, h, cfg, d_out, out_step, d_orig, orig_step)


def device(x):
    d = Dev(x)
    d.lane_bytes = x[0].nbytes
    return d


# ---- configurations --------------------------------------------------------------------------------------------------
def with_roi(cfg, roi):
    """cfg with its ROI fields replaced by roi (None: cfg itself)"""
    if roi is None:
        return cfg
    out = dataclasses.replace(cfg)
    out.preprocess = dataclasses.replace(cfg.preprocess, roiX=roi[0], roiY=roi[1], roiW=roi[2], roiH=roi[3])
    return out


def chain(lanes, options=()):
    ch = L.ProcessingChainB200(0, lanes=lanes)
    for k, v in options:
        ch.magnifier.set_option(k, v)
    return ch


def geometry(cfg, w, h, c):
    i = L.ProcessingChainB200.geometry(cfg, w, h, c)
    dw, dh = (i.out_w, i.out_h) if not i.cur_is_input else (w, h)
    return dw, dh, (i.out_channels if not i.cur_is_input else c)


def assert_same_state(m, k, tw, mode):
    """lane k of m and lane 0 of the twin hold the same temporal state"""
    if mode == O.MODE_COLOR:
        for name, lv in state_names(tw.magnifier, mode):
            assert np.array_equal(m.magnifier.get_state(name, lv)[k], tw.magnifier.get_state(name, lv)[0], equal_nan=True), (k, name)
    else:
        assert m.save_lane(k) == tw.save_lane(0), k


# ---- the check -------------------------------------------------------------------------------------------------------
def check_lanes(mode, ui, w, h, rois, steps, kind="bgr", down=1, gray=False, clip=1, options=(), entry="device", depth=3,
                split=capi.MC_SPLIT_LEFT_RIGHT, canvas=capi.MC_CANVAS_BGR, labels=False, base_roi=(0.0, 0.0, 0.5, 0.5)):
    """A len(rois)-lane chain handle, lane k with ROI override rois[k] (None: the call's base_roi), against one 1-lane twin
    per lane fed that lane's frames with its effective config.  steps: a list of per-call action lists, applied before
    that call (for submits: at submit, with earlier frames in flight): ("roi", k, roi|None), ("hold", k, on), ("reset",).
    entry: "device" (chain device calls of `clip` frames), "compose" (chain compose of BGR or NV12 sources into `canvas`)
    or "submit" (pageable chain submits of BGR frames at `depth`)."""
    lanes = len(rois)
    base = chain_cfg(mode, ui, down, base_roi, gray)
    c = 1 if kind == "gray" else 3
    m = chain(lanes, options + ((("pipeline_depth", depth),) if entry == "submit" else ()))
    over, held = list(rois), [False] * lanes
    for k, r in enumerate(over):
        if r is not None:
            m.set_lane_roi(k, r)
    twins = [chain(1, options) for _ in range(lanes)]
    ov = None
    pending = []

    def expected_geometry():
        k0 = next((k for k in range(lanes) if not held[k]), 0)
        return with_roi(base, over[k0])

    for i, acts in enumerate(steps):
        for a in acts:
            if a[0] == "roi":
                over[a[1]] = a[2]
                m.set_lane_roi(a[1], a[2])
            elif a[0] == "hold":
                held[a[1]] = a[2]
                m.magnifier.hold_lane(a[1], a[2])   # the twin is simply not fed while its lane is held
            elif a[0] == "reset":
                m.reset()
                for tw in twins:
                    tw.reset()
            elif a[0] == "save" and mode != O.MODE_COLOR:   # a lane's blob mid-run, held or not, is its twin's
                assert m.save_lane(a[1]) == twins[a[1]].save_lane(0), (i, a)
        bgr = np.stack([lane_frame(clip * i + t, k, w, h, 3) for t in range(clip) for k in range(lanes)])
        src = pack(kind, bgr)
        eff = [with_roi(base, r) for r in over]
        dw, dh, cc = geometry(expected_geometry(), w, h, c)
        v = clip * lanes
        if entry == "compose":
            cw, chh = L.MagnificationProcessor.compose_geometry(expected_geometry(), w, h, c, split)
            if labels and ov is None:
                ov = export_labels(cw, chh, split)
                m.magnifier.set_overlay(ov)
                for tw in twins:
                    tw.magnifier.set_overlay(ov)
            got = compose_call(m, kind, base, clip, w, h, src, split, canvas, cw, chh)
            assert np.array_equal(m.magnifier.lane_produced(), got[0][-1]), i
            want = [None if held[k] else compose_call(twins[k], kind, eff[k], clip, w, h, src[k::lanes], split, canvas, cw, chh)
                    for k in range(lanes)]
            compare(i, got, want, lanes, clip, held)
            continue
        out = np.full((v, dh, dw * cc), SENTINEL, np.uint8)
        orig = np.full((v, dh, dw * c if kind in ("bgr", "gray") else dw * 3), SENTINEL, np.uint8)
        if entry == "submit":
            host = np.ascontiguousarray(src)
            info = m.submit(host.ctypes.data, w, h, c, w * c, base, out.ctypes.data, dw * cc, orig.ctypes.data, orig.shape[2])
            pending.append((i, host, out, orig, info, list(held), eff))
            if len(pending) >= depth:
                finish_submit(m, twins, pending.pop(0), lanes, w, h, c)
            continue
        d_in, d_out, d_orig = device(src), Dev(out), Dev(orig)
        flags, info = call(m, kind, base, clip, w, h, d_in, d_out.ptr, dw * cc, d_orig.ptr, orig.shape[2])
        got = (flags, info, d_out.numpy(), d_orig.numpy())
        assert np.array_equal(m.magnifier.lane_produced(), flags[-1]), i
        want = []
        for k in range(lanes):
            if held[k]:
                want.append(None)
                continue
            tout, torig = out[k::lanes].copy(), orig[k::lanes].copy()
            t_in, t_out, t_orig = device(src[k::lanes]), Dev(tout), Dev(torig)
            tf, ti = call(twins[k], kind, eff[k], clip, w, h, t_in, t_out.ptr, dw * cc, t_orig.ptr, orig.shape[2])
            want.append((tf, ti, t_out.numpy(), t_orig.numpy()))
        compare(i, got, want, lanes, clip, held)
    while pending:
        finish_submit(m, twins, pending.pop(0), lanes, w, h, c)
    for k in range(lanes):
        assert_same_state(m, k, twins[k], mode)
    return m, twins


def compare(i, got, want, lanes, clip, held):
    flags, info, out, orig = got
    assert bool(info.magnified) == bool(flags.any()), i
    for k in range(lanes):
        if want[k] is None:
            assert not flags[:, k].any(), (i, k)
            assert (out[k::lanes] == SENTINEL).all(), (i, k)
            if orig is not None:
                assert (orig[k::lanes] == SENTINEL).all(), (i, k)
            continue
        tf, ti, tout, torig = want[k]
        assert np.array_equal(flags[:, k], tf[:, 0]), (i, k, flags[:, k], tf[:, 0])
        assert info_tuple(info)[:-1] == info_tuple(ti)[:-1], (i, k)
        assert np.array_equal(out[k::lanes], tout), (i, k, "out")
        if orig is not None:
            assert np.array_equal(orig[k::lanes], torig), (i, k, "orig")


def finish_submit(m, twins, item, lanes, w, h, c):
    i, host, out, orig, info, held, eff = item
    flags = m.collect()
    lane_flags = np.array(flags, bool)
    for k in range(lanes):
        if held[k]:
            assert not lane_flags[k], (i, k)
            continue
        tout, torig = np.full_like(out[k:k + 1], SENTINEL), np.full_like(orig[k:k + 1], SENTINEL)
        tw_in = np.ascontiguousarray(host[k:k + 1])
        twins[k].submit(tw_in.ctypes.data, w, h, c, w * c, eff[k], tout.ctypes.data, out.shape[2], torig.ctypes.data, orig.shape[2])
        tf = twins[k].collect()
        assert bool(lane_flags[k]) == bool(tf[0]), (i, k)
        assert np.array_equal(out[k:k + 1], tout), (i, k, "out")
        assert np.array_equal(orig[k:k + 1], torig), (i, k, "orig")


def compose_call(ch, kind, cfg, frames, w, h, src, split, fmt, cw, chh):
    """One device compose call (BGR or NV12 source) into sentinel-filled canvases -> (flags, info, canvases, None)"""
    v = len(src)
    rows = chh if fmt == capi.MC_CANVAS_BGR else chh * 3 // 2
    pitch = cw * 3 if fmt == capi.MC_CANVAS_BGR else cw
    cv = Dev(np.full((v, rows, pitch), SENTINEL, np.uint8))
    canvas = capi.McCanvas(fmt, cv.ptr, None if fmt == capi.MC_CANVAS_BGR else cv.ptr + chh * cw, pitch, rows * pitch)
    d_in = device(src)
    if kind == "nv12":
        n = w * h
        flags, info = ch.magnifier.chain_compose_nv12_device(capi.McNv12(d_in.ptr, d_in.ptr + n, w, d_in.lane_bytes), frames, w, h,
                                                             cfg, split, canvas)
    else:
        flags, info = ch.magnifier.chain_compose_device(d_in.ptr, frames, w, h, 3, w * 3, cfg, split, canvas)
    ch.magnifier.sync()
    return flags, info, cv.numpy(), None


# ---- shared with the emulation suite (tests/test_emu_lane_roi.py) ----------------------------------------------------
W, H = 96, 64
ROIS4 = [(0.0, 0.0, 0.5, 0.5), (0.5, 0.5, 0.5, 0.5), None, (0.25, 0.125, 0.5, 0.5)]
ODD = [(1 / 96, 1 / 64, 0.5, 0.5), (47 / 96, 31 / 64, 0.5, 0.5), (0.5, 0.5, 0.5, 0.5), (3 / 96, 5 / 64, 0.5, 0.5)]   # odd origins, edges


def moves(n=6):
    """one lane moved while the others run, a held lane moved while held, an override cleared"""
    s = [[] for _ in range(n)]
    s[2] = [("roi", 1, (0.125, 0.25, 0.5, 0.5)), ("hold", 3, True)]
    s[3] = [("roi", 3, (0.375, 0.0, 0.5, 0.5))]
    s[4] = [("hold", 3, False), ("roi", 0, None)]
    return s


def check_sources(kind, w=W, h=H):
    mode, ui = MODES["laplace"]
    check_lanes(mode, ui, w, h, ROIS4, moves(), kind=kind)
    if kind in ("nv12", "i420", "yv12", "yuyv"):
        check_lanes(mode, ui, w, h, ODD, moves(5), kind=kind)


def held_moves(n=7):
    """a held lane's ROI moved and moved back during the hold (no restart on release), another held lane's moved and
    cleared (a restart on release), and blobs saved while held and after the release"""
    s = [[] for _ in range(n)]
    s[1] = [("hold", 1, True), ("hold", 2, True)]
    s[2] = [("roi", 1, (0.0, 0.5, 0.5, 0.5)), ("roi", 2, (0.25, 0.25, 0.5, 0.5)), ("save", 1), ("save", 2)]
    s[3] = [("save", 1), ("save", 2), ("roi", 1, ROIS4[1])]
    s[4] = [("save", 1), ("save", 2), ("hold", 1, False), ("hold", 2, False)]
    s[5] = [("save", 1), ("save", 2)]
    s[6] = [("save", 1), ("save", 2)]
    return s


def check_modes(mname, w=W, h=H, lifecycle=True):
    mode, ui = MODES[mname]
    opts = (("color_lane_lifecycle", 1),) if mode == O.MODE_COLOR and lifecycle else ()
    check_lanes(mode, ui, w, h, ROIS4, moves(8), options=opts)
    check_lanes(mode, ui, w, h, ROIS4, held_moves(), options=opts)
    check_lanes(mode, ui, w, h, ROIS4, [[]] * 3 + [[("roi", 2, (0.5, 0.0, 0.5, 0.5))]] + [[]] * 2, clip=3, options=opts)


def check_downscale(down, w=W, h=H):
    mode, ui = MODES["laplace"]
    rois = [(0.0, 0.0, 0.75, 0.75), (0.25, 0.25, 0.75, 0.75), (0.125, 0.0, 0.75, 0.75)]
    for kind in ("bgr", "nv12"):
        check_lanes(mode, ui, w, h, rois, moves(5)[:2] + [[("roi", 1, (0.0, 0.25, 0.75, 0.75))]] + [[]] * 2, kind=kind, down=down)
    check_lanes(mode, ui, w, h, rois, [[]] * 3, kind="bgr", down=down, gray=True)


def check_clips(clip, w=W, h=H):
    mode, ui = MODES["laplace"]
    check_lanes(mode, ui, w, h, ROIS4[:3], [[], [("roi", 0, (0.5, 0.0, 0.5, 0.5))], []], clip=clip)


def check_compose(kind, fmt, w=W, h=H):
    mode, ui = MODES["laplace"]
    check_lanes(mode, ui, w, h, ROIS4, moves(5), kind=kind, entry="compose", canvas=fmt, labels=True)


def check_submits(depth, w=W, h=H):
    mode, ui = MODES["laplace"]
    check_lanes(mode, ui, w, h, ROIS4, moves(7), entry="submit", depth=depth)


def check_color_refusal(w=W, h=H):
    """Without color_lane_lifecycle, moving one Color lane's ROI is refused and changes nothing; moving every lane's at
    once is a structural reset, as before."""
    mode, ui = MODES["color"]
    base = chain_cfg(mode, ui, 1, (0.0, 0.0, 0.5, 0.5))
    a, b = chain(3), chain(3)

    def run(ch, t):
        bgr = np.stack([lane_frame(t, k, w, h, 3) for k in range(3)])
        d_in, out = device(bgr), Dev(np.full((3, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        flags, info = ch.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
        ch.magnifier.sync()
        return flags, out.numpy()

    for t in range(3):
        run(a, t), run(b, t)
    launches = a.magnifier.launch_count
    a.set_lane_roi(1, (0.5, 0.5, 0.5, 0.5))
    with pytest.raises(capi.MagcoreError) as e:
        run(a, 3)
    assert e.value.status == capi.MC_ERR_UNSUPPORTED
    assert a.magnifier.launch_count == launches
    a.set_lane_roi(1, None)
    for t in range(3, 6):
        fa, oa = run(a, t)
        fb, ob = run(b, t)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob), t
    for k in range(3):
        a.set_lane_roi(k, (0.25, 0.25, 0.5, 0.5))
        b.set_lane_roi(k, (0.25, 0.25, 0.5, 0.5))
    for t in range(6, 8):
        fa, oa = run(a, t)
        fb, ob = run(b, t)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob), t


def check_unequal_sizes(w=W, h=H):
    """Lanes whose crops differ in pixel size are refused before any copy or launch, naming the lane; buffers, state and
    launch count stay as they were.  A held lane is not checked until it runs."""
    mode, ui = MODES["laplace"]
    base = chain_cfg(mode, ui, 1, (0.0, 0.0, 0.5, 0.5))
    m, ref = chain(3), chain(3)
    bgr = [np.stack([lane_frame(t, k, w, h, 3) for k in range(3)]) for t in range(4)]

    def run(ch, t):
        d_in, out = device(bgr[t]), Dev(np.full((3, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        flags, _ = ch.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
        ch.magnifier.sync()
        return flags, out

    run(m, 0), run(ref, 0)
    blobs, launches = [m.save_lane(k) for k in range(3)], m.magnifier.launch_count
    m.set_lane_roi(2, (0.25, 0.25, 0.75, 0.5))
    out = Dev(np.full((3, h // 2, w // 2 * 3), SENTINEL, np.uint8))
    d_in = device(bgr[1])
    with pytest.raises(capi.MagcoreError) as e:
        m.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
    assert e.value.status == capi.MC_ERR_INVALID and "lane 2" in capi.lib().mc_last_error(m.magnifier._h).decode()
    assert (out.numpy() == SENTINEL).all() and m.magnifier.launch_count == launches
    assert [m.save_lane(k) for k in range(3)] == blobs
    m.magnifier.hold_lane(2, True)
    ref.magnifier.hold_lane(2, True)
    fm, om = run(m, 1)
    fr, orf = run(ref, 1)
    assert np.array_equal(fm, fr) and np.array_equal(om.numpy(), orf.numpy())
    m.magnifier.hold_lane(2, False)
    with pytest.raises(capi.MagcoreError):
        run(m, 2)


def check_reset_and_clear(w=W, h=H):
    """Overrides survive reset(); a handle whose overrides were set and cleared equals a fresh handle, launch count
    included."""
    mode, ui = MODES["laplace"]
    steps = [[], [], [("reset",)], [], [("roi", 1, None)], []]
    check_lanes(mode, ui, w, h, ROIS4, steps)
    base = chain_cfg(mode, ui, 1, (0.0, 0.0, 0.5, 0.5))
    a, b = chain(4), chain(4)
    for k, r in enumerate(ROIS4):
        a.set_lane_roi(k, r)

    def run(ch, t):
        bgr = np.stack([lane_frame(t, k, w, h, 3) for k in range(4)])
        d_in, out = device(bgr), Dev(np.full((4, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        flags, _ = ch.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
        ch.magnifier.sync()
        return flags, out.numpy()

    for t in range(3):
        run(a, t)
    for k in range(4):
        a.set_lane_roi(k, None)
    a.reset()
    la, lb = a.magnifier.launch_count, b.magnifier.launch_count
    for t in range(5):
        fa, oa = run(a, t)
        fb, ob = run(b, t)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob), t
    assert a.magnifier.launch_count - la == b.magnifier.launch_count - lb
    assert [a.save_lane(k) for k in range(4)] == [b.save_lane(k) for k in range(4)]


def check_save_load(w=W, h=H):
    """A blob carries its lane's own ROI: it loads into a lane of a handle without state (which then restarts the lane
    when its ROI differs, as the source lane's twin would) and into a lane whose fingerprint is the same; a lane whose
    ROI fingerprint differs refuses it."""
    mode, ui = MODES["laplace"]
    base = chain_cfg(mode, ui, 1, (0.0, 0.0, 0.5, 0.5))
    ra, rb = (0.5, 0.5, 0.5, 0.5), (0.25, 0.0, 0.5, 0.5)

    def run(ch, t, lanes, cfg=base):
        bgr = np.stack([lane_frame(t, k, w, h, 3) for k in range(lanes)])
        d_in, out = device(bgr), Dev(np.full((lanes, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        flags, _ = ch.process_device(d_in.ptr, 1, w, h, 3, w * 3, cfg, out.ptr, w // 2 * 3)
        ch.magnifier.sync()
        return flags, out.numpy()

    src = chain(2)
    src.set_lane_roi(1, ra)
    for t in range(3):
        run(src, t, 2)
    blob = src.save_lane(1)
    # refused: lane 0 of src runs at the call's ROI
    with pytest.raises(capi.MagcoreError):
        src.load_lane(0, blob)
    # a fresh 2-lane handle takes the blob into lane 0, whose override is ra: it continues as src's lane 1
    dst = chain(2)
    dst.set_lane_roi(0, ra)
    dst.set_lane_roi(1, rb)
    dst.load_lane(0, blob)
    twin = chain(1)
    twin.load_lane(0, blob)
    for t in range(3, 6):
        bgr = np.stack([lane_frame(t, 1, w, h, 3), lane_frame(t, 0, w, h, 3)])
        d_in, out = device(bgr), Dev(np.full((2, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        fd, _ = dst.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
        dst.magnifier.sync()
        t_in, t_out = device(bgr[:1]), Dev(np.full((1, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        ft, _ = twin.process_device(t_in.ptr, 1, w, h, 3, w * 3, with_roi(base, ra), t_out.ptr, w // 2 * 3)
        twin.magnifier.sync()
        s_in, s_out = device(np.stack([lane_frame(t, 0, w, h, 3), lane_frame(t, 1, w, h, 3)])), \
            Dev(np.full((2, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        fs, _ = src.process_device(s_in.ptr, 1, w, h, 3, w * 3, base, s_out.ptr, w // 2 * 3)
        src.magnifier.sync()
        assert fd[0, 0] and ft[0, 0] and fs[0, 1]
        assert np.array_equal(out.numpy()[0], t_out.numpy()[0]) and np.array_equal(out.numpy()[0], s_out.numpy()[1]), t
    assert dst.save_lane(0) == src.save_lane(1) == twin.save_lane(0)
    # loaded into a fresh handle whose lane runs at another ROI: that lane restarts, as the source lane's twin would
    other = chain(2)
    other.set_lane_roi(1, rb)
    other.load_lane(1, blob)
    twin = chain(1)
    twin.load_lane(0, blob)
    for t in range(6, 8):
        bgr = np.stack([lane_frame(t, 0, w, h, 3), lane_frame(t, 1, w, h, 3)])
        d_in, out = device(bgr), Dev(np.full((2, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        fo, _ = other.process_device(d_in.ptr, 1, w, h, 3, w * 3, base, out.ptr, w // 2 * 3)
        other.magnifier.sync()
        t_in, t_out = device(bgr[1:]), Dev(np.full((1, h // 2, w // 2 * 3), SENTINEL, np.uint8))
        ft, _ = twin.process_device(t_in.ptr, 1, w, h, 3, w * 3, with_roi(base, rb), t_out.ptr, w // 2 * 3)
        twin.magnifier.sync()
        assert fo[0, 1] == ft[0, 0] and np.array_equal(out.numpy()[1], t_out.numpy()[0]), t
    assert other.save_lane(1) == twin.save_lane(0)


def check_magnifier_only(w=W, h=H):
    """mc_process does not crop: a lane's ROI override only enters its fingerprint, so moving it restarts that lane."""
    mode, ui = MODES["laplace"]
    cfg = chain_cfg(mode, ui)
    m = L.MagnificationProcessor(0, lanes=3)
    twins = [L.MagnificationProcessor(0) for _ in range(3)]
    rois = [None, None, None]
    for t in range(6):
        if t == 2:
            rois[1] = (0.1, 0.2, 0.3, 0.4)
            m.set_lane_roi(1, rois[1])
        if t == 4:
            rois[1] = None
            m.set_lane_roi(1, None)
        f = np.stack([lane_frame(t, k, w, h, 3) for k in range(3)])
        out = np.full_like(f, SENTINEL)
        prod = m.process_host(f.ctypes.data, w, h, 3, w * 3, cfg, out.ctypes.data, w * 3)
        flags = m.lane_produced()
        for k in range(3):
            p, o = twins[k].process_image(f[k], with_roi(cfg, rois[k]))
            assert bool(flags[k]) == bool(p), (t, k)
            if p:
                assert np.array_equal(out[k], o), (t, k)
        assert bool(prod) == bool(flags.any())


def check_errors():
    lib = capi.lib()
    m = L.MagnificationProcessor(0, lanes=2)
    roi = (C.c_float * 4)(0, 0, 1, 1)
    for bad in (-1, 2):
        assert lib.mc_set_lane_roi(m._h, bad, roi) == capi.MC_ERR_INVALID
    assert lib.mc_set_lane_roi(None, 0, roi) == capi.MC_ERR_INVALID
    assert lib.mc_set_lane_roi(m._h, 1, None) == capi.MC_OK
    for bad in ((0.0, 0.0, 1.0), (0.0, 0.0, 1.0, 1.0, 0.0)):
        with pytest.raises(ValueError):
            m.set_lane_roi(0, bad)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", SOURCES)
def test_every_source(kind):
    check_sources(kind)


@pytest.mark.parametrize("mname", ["laplace", "phase", "color"])
def test_modes(mname):
    check_modes(mname)


def test_color_without_lane_lifecycle():
    check_color_refusal()


@pytest.mark.parametrize("down", [1, 2, 3])
def test_downscale(down):
    check_downscale(down)


@pytest.mark.parametrize("clip", [1, 3, 16])
def test_clips(clip):
    check_clips(clip)


@pytest.mark.parametrize("kind,fmt", [("bgr", capi.MC_CANVAS_BGR), ("nv12", capi.MC_CANVAS_NV12), ("bgr", capi.MC_CANVAS_I420)])
def test_compose(kind, fmt):
    check_compose(kind, fmt)


@pytest.mark.parametrize("depth", [1, 3, 5])
def test_submits(depth):
    check_submits(depth)


def test_unequal_sizes_refused():
    check_unequal_sizes()


def test_reset_keeps_and_none_clears():
    check_reset_and_clear()


def test_save_and_load_between_lanes_with_different_rois():
    check_save_load()


def test_magnifier_only_calls():
    check_magnifier_only()


def test_errors():
    check_errors()


@pytest.mark.skipif(EMU, reason="4K frames are too slow for the CPU emulation")
def test_64_lanes_of_4k_crops_against_the_reference():
    """64 lanes of 4K frames, each cropped to its own 1920 x 1080 window, Laplace at 6 levels: lanes 0 and 63 equal their
    1-lane twins and are within 1 LSB of the compiled reference run with that lane's ROI."""
    from test_gpu_long_runs import RefCore, u8_diff
    from lvm_b200.synth import synth_frame
    w, h, lanes, n = 3840, 2160, 64, 3
    mode, ui = O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 6)
    cfg = chain_cfg(mode, ui, 1, (0.0, 0.0, 0.5, 0.5))
    rois = [((k % 8) * 240 / w, (k // 8) * 135 / h, 0.5, 0.5) for k in range(lanes)]
    m = chain(lanes)
    for k, r in enumerate(rois):
        m.set_lane_roi(k, r)
    import torch
    base = [torch.from_numpy(synth_frame(t, w, h, 3)).cuda() for t in range(n)]
    out = torch.empty((lanes, 1080, 1920 * 3), dtype=torch.uint8, device="cuda")
    twins = {}
    for t in range(n):
        frames = base[t].unsqueeze(0).expand(lanes, h, w, 3).contiguous()
        flags, info = m.process_device(frames.data_ptr(), 1, w, h, 3, w * 3, cfg, out.data_ptr(), 1920 * 3)
        m.magnifier.sync()
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        for k in (0, lanes - 1):
            tw, ref = twins.setdefault(k, (chain(1), RefCore(mode)))
            eff = with_roi(cfg, rois[k])
            f = synth_frame(t, w, h, 3)
            tin, tout = device(f[None]), Dev(np.full((1, 1080, 1920 * 3), SENTINEL, np.uint8))
            tf, _ = tw.process_device(tin.ptr, 1, w, h, 3, w * 3, eff, tout.ptr, 1920 * 3)
            tw.magnifier.sync()
            assert bool(tf[0, 0]) == bool(flags[0, k]) and np.array_equal(got[k], tout.numpy()[0]), (t, k)
            x, y = round(rois[k][0] * w), round(rois[k][1] * h)
            crop = np.ascontiguousarray(f[y:y + 1080, x:x + 1920])
            ocfg = O.ProcessorConfig(magnification=O.to_params(mode, 20, 50.0, 0.4, 3.0, 0, 6, 30.0))
            rp, rout = ref.run(crop, ocfg)
            if flags[0, k]:
                assert rp and int(u8_diff(got[k].reshape(1080, 1920, 3), rout).max()) <= 1, (t, k)

