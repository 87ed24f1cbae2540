"""Clips (mc_process_clip / mc_process_clip_device): T consecutive frames in one call must equal, bit for bit, the same
frames fed one frame call at a time to a handle with the same options — u8 outputs, produced flags, mc_lane_produced
and the temporal state planes afterwards."""
import ctypes as C

import numpy as np
import pytest

from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_lanes import (COLOR_UI, LAPLACE_UI, PHASE_UI, SENTINEL, assert_lane_state_equal, lane_frame, proc,
                            process_raw, single_run, state_names)

U8P = C.POINTER(C.c_uint8)


def clip_frames(t0, n, lanes, w, h, c):
    """[n, lanes, H, W(, C)]: frames t0 .. t0+n-1 of every lane."""
    return np.stack([np.stack([lane_frame(t, k, w, h, c) for k in range(lanes)]) for t in range(t0, t0 + n)])


def geom(frames):
    """[T, lanes, H, W(, C)] -> (T, w, h, c)"""
    return frames.shape[0], frames.shape[3], frames.shape[2], 1 if frames.ndim == 4 else frames.shape[4]


def run_clip(p, frames, cfg):
    """One mc_process_clip call into a sentinel-filled buffer -> (flags u8 [T, lanes], out)."""
    n, w, h, c = geom(frames)
    out = np.full_like(frames, SENTINEL)
    flags = np.zeros((n, p.lanes), np.uint8)
    prm = _to_mc(cfg)
    p._check(p._lib.mc_process_clip(p._h, frames.ctypes.data, n, w, h, c, w * c, C.byref(prm), out.ctypes.data, w * c,
                                    flags.ctypes.data_as(U8P)))
    return flags, out


def run_frames(p, frames, cfg):
    """The same frames, one mc_process call each (sentinel-filled buffers) -> (flags u8 [T, lanes], out)."""
    flags, outs = [], []
    for f in frames:
        _, out, fl = process_raw(p, f, cfg)
        flags.append(fl.astype(np.uint8))
        outs.append(out)
    return np.stack(flags), np.stack(outs)


def assert_states_equal(a, b, mode):
    names = state_names(b, mode)
    assert names == state_names(a, mode)
    for n, l in names:
        assert np.array_equal(a.get_state(n, l), b.get_state(n, l)), (n, l)
    return names


def check_clip(mode, ui, w, h, c, steps, lanes=1, options=()):
    """Two handles with the same options take the same frames: `steps` is a list of
        ("clip", n)    one clip of n frames on the first handle,
        ("frames", n)  n frame calls on it,
        ("ui", ui)     new parameters from here on,   ("size", (w, h))  a new frame size,   ("reset", None)  mc_reset;
    the second handle always takes frame calls.  After every step the flags, the u8 outputs (the sentinel where a frame
    did not produce), mc_lane_produced and the state planes are equal.  -> the first handle's flags per step."""
    cfg, _ = make_cfgs(mode, *ui)
    a, b = proc(lanes, options), proc(lanes, options)
    t, got = 0, []
    for i, (kind, arg) in enumerate(steps):
        if kind == "ui":
            cfg, _ = make_cfgs(mode, *arg)
            continue
        if kind == "size":
            w, h = arg
            continue
        if kind == "reset":
            a.reset()
            b.reset()
            continue
        fr = clip_frames(t, arg, lanes, w, h, c)
        fa, oa = run_clip(a, fr, cfg) if kind == "clip" else run_frames(a, fr, cfg)
        fb, ob = run_frames(b, fr, cfg)
        assert np.array_equal(fa, fb), (i, fa.tolist(), fb.tolist())
        assert np.array_equal(oa, ob), i
        assert np.array_equal(a.lane_produced(), b.lane_produced()), i
        assert_states_equal(a, b, mode)
        got.append(fa)
        t += arg
    a.close()
    b.close()
    return got


def check_lanes_clip(mode, ui, w, h, c, lanes=4, restart=2, hold=1, clips=(3, 4, 2), options=()):
    """Clip A runs every lane; before clip B lane `restart` is restarted and lane `hold` held; the hold is released before
    clip C.  Each lane equals its own 1-lane processor fed its frames one call at a time: restarted where the lane was,
    not fed at all while it was held (flags 0 and its bytes of out untouched there)."""
    cfg, _ = make_cfgs(mode, *ui)
    m = proc(lanes, options)
    flags, outs, t = [], [], 0
    for i, n in enumerate(clips):
        if i == 1:
            m.restart_lane(restart)
            m.hold_lane(hold)
        if i == 2:
            m.hold_lane(hold, False)
        f, o = run_clip(m, clip_frames(t, n, lanes, w, h, c), cfg)
        flags.append(f)
        outs.append(o)
        t += n
    flags, outs = np.concatenate(flags), np.concatenate(outs)
    b0, b1 = clips[0], clips[0] + clips[1]
    for k in range(lanes):
        if k == restart:
            runs = [list(range(b0)), list(range(b0, t))]
        elif k == hold:
            runs = [list(range(b0)) + list(range(b1, t))]
            assert not flags[b0:b1, k].any() and (outs[b0:b1, k] == SENTINEL).all()
        else:
            runs = [list(range(t))]
        for ts in runs:
            ref, sp = single_run([lane_frame(tt, k, w, h, c) for tt in ts], cfg, options)
            for tt, (sprod, sout) in zip(ts, ref):
                assert bool(flags[tt, k]) == bool(sprod), (k, tt)
                if sprod:
                    assert np.array_equal(outs[tt, k], sout), (k, tt)
                else:
                    assert (outs[tt, k] == SENTINEL).all(), (k, tt)
        assert_lane_state_equal(m, k, sp, mode)
    assert np.array_equal(m.lane_produced(), flags[-1].astype(bool))
    m.close()


def laplace_ui(levels):
    return LAPLACE_UI[:5] + (levels,)


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("levels", [1, 2, 3, 4, 6])
@pytest.mark.parametrize("w,h", [(240, 135), (83, 45), (30, 17)])
def test_laplace_clip_one_lane(w, h, levels, c):
    """T = 1, 2, 5, 16 on a fresh handle (its first frame inside the clip), then a second clip on the continuing one."""
    for n in (1, 2, 5, 16):
        check_clip(O.MODE_LAPLACE, laplace_ui(levels), w, h, c, [("clip", n), ("clip", n)])


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_1080p(c):
    check_clip(O.MODE_LAPLACE, laplace_ui(6), 1920, 1080, c, [("clip", 8), ("clip", 8)])


def test_laplace_clip_interleaves_with_frame_calls():
    check_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, [("frames", 3), ("clip", 4), ("frames", 2), ("clip", 5)])


def test_laplace_clip_parameter_change_between_clips():
    """amplification, cutoffs and chroma are not structural: the state carries over"""
    check_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, [("clip", 4), ("ui", (35, 30.0, 0.8, 2.0, 70, 4)), ("clip", 4)])


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_size_change_at_clip_start(c):
    check_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, c, [("clip", 3), ("size", (97, 61)), ("clip", 4), ("size", (131, 75)),
                                                         ("clip", 2)])


def test_laplace_clip_reset_between_clips():
    check_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, [("clip", 3), ("reset", None), ("clip", 4), ("frames", 1)])


@pytest.mark.parametrize("options", [(("use_tma", 0),), (("use_tma", 1),), (("egress_strip", 0),), (("egress_strip", 1),)])
@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_options(options, c):
    """400 x 300: level 1 has interior tiles as well as border tiles"""
    check_clip(O.MODE_LAPLACE, laplace_ui(5), 400, 300, c, [("clip", 5), ("clip", 3)], options=options)


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_faithful_level0(c):
    levels = 4
    cfg_levels = laplace_ui(levels)
    got = check_clip(O.MODE_LAPLACE, cfg_levels, 131, 75, c, [("clip", 4), ("clip", 3)], options=(("faithful_level0", 1),))
    assert len(got) == 2
    p = proc(1, (("faithful_level0", 1),))
    run_clip(p, clip_frames(0, 2, 1, 131, 75, c), make_cfgs(O.MODE_LAPLACE, *cfg_levels)[0])
    names = state_names(p, O.MODE_LAPLACE)
    assert ("lowpassHi", 0) in names and ("lowpassLo", levels) in names   # the level-0 and residual planes were compared
    p.close()


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_analysis_only(c):
    """only the handle's first frame is produced; the state equals the sequential state"""
    got = check_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, c, [("clip", 4), ("clip", 3)], options=(("analysis_only", 1),))
    assert got[0][:, 0].tolist() == [1, 0, 0, 0] and not got[1].any()


def test_laplace_clip_lane_groups():
    check_clip(O.MODE_LAPLACE, LAPLACE_UI, 83, 45, 3, [("clip", 3), ("clip", 2)], lanes=16, options=(("lane_groups", 2),))


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_lanes_restart_and_hold(c):
    check_lanes_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, c)


def test_laplace_clip_lanes_faithful_level0():
    check_lanes_clip(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, options=(("faithful_level0", 1),))


def test_laplace_clip_profile_names_the_kernel():
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    p = proc(1, (("profile_kernels", 1),))
    run_clip(p, clip_frames(0, 3, 1, 131, 75, 3), cfg)
    prof = p.profile_read()
    assert prof[("level_clip", 1)][0] == 1 and ("level", 1) not in prof
    p.close()


def test_phase_clip():
    """the first clip holds Phase's passthrough first frame"""
    got = check_clip(O.MODE_PHASE, PHASE_UI, 120, 90, 3, [("clip", 4), ("clip", 3)])
    assert got[0][:, 0].tolist() == [0, 1, 1, 1]


def test_color_clip():
    """the first clip holds Color's warm-up"""
    got = check_clip(O.MODE_COLOR, COLOR_UI, 120, 90, 3, [("clip", 4), ("clip", 4)])
    assert got[0][0, 0] == 0 and got[1].all()


@pytest.mark.parametrize("mode,ui", [(O.MODE_LAPLACE, LAPLACE_UI), (O.MODE_PHASE, PHASE_UI)])
def test_host_clip_matches_device_clip(mode, ui):
    """mc_process_clip with pageable and with pinned buffers equals mc_process_clip_device; frames that did not produce
    keep the sentinel, and process_clip fills them with their inputs."""
    torch = pytest.importorskip("torch")
    cfg, _ = make_cfgs(mode, *ui)
    w, h, c = 131, 75, 3
    frames = clip_frames(0, 5, 1, w, h, c)
    n = frames.shape[0]

    dev = proc()
    d_in = torch.from_numpy(frames).cuda()
    d_out = torch.full_like(d_in, SENTINEL)
    torch.cuda.synchronize()
    f_dev = dev.process_clip_device(d_in.data_ptr(), n, w, h, c, w * c, cfg, d_out.data_ptr(), w * c)
    dev.sync()
    o_dev = d_out.cpu().numpy()

    pageable = proc()
    f_pg, o_pg = run_clip(pageable, frames, cfg)

    pinned = proc()
    pin_in = torch.from_numpy(frames).pin_memory()
    pin_out = torch.full(frames.shape, SENTINEL, dtype=torch.uint8).pin_memory()
    f_pin = np.zeros((n, 1), np.uint8)
    prm = _to_mc(cfg)
    pinned._check(pinned._lib.mc_process_clip(pinned._h, pin_in.data_ptr(), n, w, h, c, w * c, C.byref(prm), pin_out.data_ptr(),
                                              w * c, f_pin.ctypes.data_as(U8P)))
    o_pin = pin_out.numpy()

    assert np.array_equal(f_dev, f_pg.astype(bool)) and np.array_equal(f_pg, f_pin)
    assert np.array_equal(o_dev, o_pg) and np.array_equal(o_pg, o_pin)
    for t in range(n):
        if not f_pg[t, 0]:
            assert (o_pg[t] == SENTINEL).all()
    if mode == O.MODE_PHASE:
        assert not f_pg[0, 0] and f_pg[1:, 0].all()

    filled = proc()
    f_py, o_py = filled.process_clip(frames[:, 0], cfg)
    assert o_py.shape == frames[:, 0].shape
    assert np.array_equal(f_py, f_pg.astype(bool))
    for t in range(n):
        assert np.array_equal(o_py[t], o_pg[t, 0] if f_pg[t, 0] else frames[t, 0]), t
    for p in (dev, pageable, pinned, filled):
        p.close()


def test_process_clip_multi_lane_shape():
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    frames = clip_frames(0, 3, 2, 83, 45, 1)
    p = proc(2)
    flags, out = p.process_clip(frames, cfg)
    assert flags.shape == (3, 2) and flags.all() and out.shape == frames.shape
    with pytest.raises(ValueError):
        p.process_clip(frames[:, 0], cfg)
    p.close()


def test_clip_bad_arguments_leave_state_untouched():
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    w, h, c, lanes = 83, 45, 3, 2
    a, b = proc(lanes), proc(lanes)
    warm = clip_frames(0, 3, lanes, w, h, c)
    run_clip(a, warm, cfg)
    run_frames(b, warm, cfg)
    fr = clip_frames(3, 2, lanes, w, h, c)
    out = np.full_like(fr, SENTINEL)
    flags = np.zeros((2, lanes), np.uint8)
    prm = _to_mc(cfg)
    lib = a._lib
    big = capi.MC_MAX_LANES // lanes + 1
    for fn in (lib.mc_process_clip, lib.mc_process_clip_device):
        for n, fl in ((0, flags), (-1, flags), (big, flags), (2, None)):
            st = fn(a._h, fr.ctypes.data, n, w, h, c, w * c, C.byref(prm), out.ctypes.data, w * c,
                    None if fl is None else fl.ctypes.data_as(U8P))
            assert st == capi.MC_ERR_INVALID, (fn, n)
    assert (out == SENTINEL).all()
    # frames of mc_submit in flight: refused; the submitted frame itself runs
    sub_out = np.empty_like(fr[0])
    a.submit(fr[0].ctypes.data, w, h, c, w * c, cfg, sub_out.ctypes.data, w * c)
    st = lib.mc_process_clip(a._h, fr.ctypes.data, 2, w, h, c, w * c, C.byref(prm), out.ctypes.data, w * c,
                             flags.ctypes.data_as(U8P))
    assert st == capi.MC_ERR_INVALID
    assert a.collect()
    _, ref, _ = process_raw(b, fr[0], cfg)
    assert np.array_equal(sub_out, ref)
    assert_states_equal(a, b, O.MODE_LAPLACE)
    # the next frame call continues from the unchanged state
    _, oa, _ = process_raw(a, fr[1], cfg)
    _, ob, _ = process_raw(b, fr[1], cfg)
    assert np.array_equal(oa, ob)
    assert_states_equal(a, b, O.MODE_LAPLACE)
    a.close()
    b.close()
