"""Phase (Riesz) clips: mc_process_clip runs a Phase clip as one launch set with the temporally batched k_riesz_phase_clip.
T consecutive frames in one call must equal, bit for bit, the same frames fed one frame call at a time: u8 outputs (the
sentinel where a frame did not produce), produced flags, mc_lane_produced and every Phase state plane afterwards."""
import ctypes as C

import numpy as np
import pytest

from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_clip import U8P, check_clip, check_lanes_clip, clip_frames, run_clip, run_frames
from test_gpu_lanes import PHASE_UI, SENTINEL, proc
from lvm_b200.processor import _to_mc

# every state plane of a Phase handle (mc_get_state names)
ALL_STATES = ("old.lowpass", "old.rx", "old.ry", "phase.c", "phase.s", "lo.r0.c", "lo.r0.s", "lo.r1.c", "lo.r1.s",
              "hi.r0.c", "hi.r0.s", "hi.r1.c", "hi.r1.s")


def phase_ui(levels=3, amplification=50, wavelength=50.0, low=0.4, high=3.0):
    return (amplification, wavelength, low, high, 0, levels)


def all_state_names(p):
    return [(n, l) for n in ALL_STATES for l in range(9) if p.state_dims(n, l)[0]]


def assert_all_states_equal(a, b, lanes=None):
    """every Phase state plane of `a` equals `b`'s (only the given lanes when `lanes` is set)"""
    names = all_state_names(b)
    assert names == all_state_names(a)
    for n, l in names:
        sa, sb = a.get_state(n, l), b.get_state(n, l)
        if lanes is not None:
            sa, sb = sa[list(lanes)], sb[list(lanes)]
        assert np.array_equal(sa, sb), (n, l)
    return names


def check_events(ui, w, h, steps, lanes=1, c=3, options=(), state_lanes=None, final_all=False):
    """Two handles with the same options take the same frames and the same lane events: `steps` is a list of
        ("clip", n), ("frames", n), ("ui", ui), ("hold", (lane, on)), ("restart", lane), ("reset", None);
    the first handle takes the "clip" steps as clips, the second always frame calls.  After every frame step the flags,
    the u8 outputs, mc_lane_produced and every state plane (of `state_lanes`, or all lanes) are equal; with final_all,
    every lane's state planes after the last step."""
    cfg, _ = make_cfgs(O.MODE_PHASE, *ui)
    a, b = proc(lanes, options), proc(lanes, options)
    t, got = 0, []
    for i, (kind, arg) in enumerate(steps):
        if kind == "ui":
            cfg, _ = make_cfgs(O.MODE_PHASE, *arg)
        elif kind == "hold":
            for p in (a, b):
                p.hold_lane(*arg)
        elif kind == "restart":
            for p in (a, b):
                p.restart_lane(arg)
        elif kind == "reset":
            for p in (a, b):
                p.reset()
        else:
            fr = clip_frames(t, arg, lanes, w, h, c)
            fa, oa = run_clip(a, fr, cfg) if kind == "clip" else run_frames(a, fr, cfg)
            fb, ob = run_frames(b, fr, cfg)
            assert np.array_equal(fa, fb), (i, fa.tolist(), fb.tolist())
            assert np.array_equal(oa, ob), i
            assert np.array_equal(a.lane_produced(), b.lane_produced()), i
            assert_all_states_equal(a, b, state_lanes)
            got.append(fa)
            t += arg
    if final_all:
        assert_all_states_equal(a, b)
    a.close()
    b.close()
    return got


pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("levels", [1, 2, 3, 6, 9])
@pytest.mark.parametrize("w,h", [(131, 75), (83, 45), (30, 17)])
def test_phase_clip_one_lane(w, h, levels):
    """T = 1, 2, 5, 16 on a fresh handle (its passthrough first frame inside the clip), then on the continuing one;
    widths that are not multiples of 8 give filter2D tail columns; 9 levels are clamped"""
    for n in (1, 2, 5, 16):
        got = check_clip(O.MODE_PHASE, phase_ui(levels), w, h, 3, [("clip", n), ("clip", n)])
        assert got[0][0, 0] == 0 and got[0][1:].all() and got[1].all()


def test_phase_clip_every_state_plane():
    check_events(phase_ui(4), 131, 75, [("clip", 5), ("clip", 3), ("frames", 2), ("clip", 4)])


def test_phase_clip_7x9():
    check_clip(O.MODE_PHASE, phase_ui(3), 7, 9, 3, [("clip", 3), ("clip", 5)])


def test_phase_clip_1080p():
    check_clip(O.MODE_PHASE, phase_ui(6), 1920, 1080, 3, [("clip", 8), ("clip", 8)])


def test_phase_clip_interleaves_with_frame_calls():
    check_clip(O.MODE_PHASE, PHASE_UI, 131, 75, 3, [("frames", 3), ("clip", 4), ("frames", 2), ("clip", 5)])


def test_phase_clip_amplification_and_wavelength_change_between_clips():
    """not cutoffs: the state carries over"""
    check_events(PHASE_UI, 131, 75, [("clip", 4), ("ui", phase_ui(3, 35, 30.0)), ("clip", 4), ("ui", phase_ui(3, 80, 70.0)),
                                     ("clip", 3)])


def test_phase_clip_cutoff_change_between_clips():
    """the filters are redesigned at the clip's first frame, whose prior is that frame itself"""
    check_events(PHASE_UI, 131, 75, [("clip", 4), ("ui", phase_ui(3, low=0.6)), ("clip", 4), ("ui", phase_ui(3, high=2.5)),
                                     ("clip", 3), ("ui", phase_ui(3, low=0.5, high=2.0)), ("frames", 2), ("clip", 2)])


def test_phase_clip_cutoff_change_while_held():
    """a cutoff change at the start of a clip in which a lane is held: that lane restarts on release (its first clip
    frame passes through).  The lanes that were never held are compared throughout, every lane once it has restarted."""
    steps = [("clip", 3), ("hold", (1, True)), ("ui", phase_ui(3, low=0.6)), ("clip", 4), ("hold", (1, False)), ("clip", 3)]
    got = check_events(PHASE_UI, 120, 90, steps, lanes=3, state_lanes=(0, 2), final_all=True)
    assert not got[1][:, 1].any()
    assert got[2][0].tolist() == [1, 0, 1] and got[2][1:].all()


@pytest.mark.parametrize("size", [(97, 61), (64, 40)])
def test_phase_clip_size_change_and_reset(size):
    check_clip(O.MODE_PHASE, PHASE_UI, 131, 75, 3, [("clip", 3), ("size", size), ("clip", 4), ("reset", None), ("clip", 2),
                                                    ("size", (131, 75)), ("clip", 3)])


@pytest.mark.parametrize("use_tma", [0, 1])
def test_phase_clip_use_tma(use_tma):
    """400 x 300: every band level has interior tiles (TMA windows) as well as border tiles (reflected loads)"""
    check_events(phase_ui(4), 400, 300, [("clip", 5), ("clip", 3)], options=(("use_tma", use_tma),))


def test_phase_clip_use_tma_same_bits():
    cfg, _ = make_cfgs(O.MODE_PHASE, *phase_ui(4))
    fr = clip_frames(0, 6, 1, 400, 300, 3)
    a, b = proc(1, (("use_tma", 1),)), proc(1, (("use_tma", 0),))
    fa, oa = run_clip(a, fr, cfg)
    fb, ob = run_clip(b, fr, cfg)
    assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
    assert_all_states_equal(a, b)
    a.close()
    b.close()


def test_phase_clip_analysis_only():
    """state only: every flag 0, the state equals the frame calls'"""
    got = check_events(PHASE_UI, 131, 75, [("clip", 4), ("clip", 3)], options=(("analysis_only", 1),))
    assert not any(g.any() for g in got)


def test_phase_clip_keep_float_output():
    """the tap holds the clip's last frame, as after the last frame call"""
    cfg, _ = make_cfgs(O.MODE_PHASE, *PHASE_UI)
    w, h, c, lanes = 131, 75, 3, 2
    a, b = proc(lanes, (("keep_float_output", 1),)), proc(lanes, (("keep_float_output", 1),))
    t = 0
    for n in (4, 3):
        fr = clip_frames(t, n, lanes, w, h, c)
        run_clip(a, fr, cfg)
        run_frames(b, fr, cfg)
        assert np.array_equal(a.float_output(w, h, c), b.float_output(w, h, c))
        t += n
    a.close()
    b.close()


def test_phase_clip_lanes_restart_and_hold():
    check_lanes_clip(O.MODE_PHASE, PHASE_UI, 131, 75, 3)


def test_phase_clip_lanes_every_state_plane():
    check_events(PHASE_UI, 83, 45, [("clip", 3), ("restart", 2), ("hold", (1, True)), ("clip", 4), ("hold", (1, False)),
                                    ("clip", 2), ("restart", 0), ("clip", 3)], lanes=4)


EDGE = [
    ("alpha 0", phase_ui(3, amplification=0)),
    ("threshold pi", phase_ui(3, wavelength=0.0)),
    ("threshold 0", phase_ui(3, wavelength=100.0)),
    ("low 0 Hz", phase_ui(3, low=0.0)),
    ("high = Nyquist", phase_ui(3, high=15.0)),
    ("high > Nyquist", phase_ui(3, high=20.0)),
]


@pytest.mark.parametrize("name,ui", EDGE, ids=[e[0] for e in EDGE])
def test_phase_clip_edge_params(name, ui):
    check_events(ui, 96, 64, [("clip", 4), ("clip", 3), ("frames", 1), ("clip", 2)])


def test_phase_clip_flat_and_letterboxed_content():
    """flat rows and columns (black bars, a flat frame) give NaN amplitudes there, shown white as by OpenCV"""
    cfg, _ = make_cfgs(O.MODE_PHASE, *PHASE_UI)
    w, h, c = 131, 75, 3
    fr = clip_frames(0, 7, 1, w, h, c)
    fr[:, :, :12] = 0          # letterbox bars
    fr[:, :, -12:] = 0
    fr[:, :, :, :9] = 16       # pillarbox bar
    fr[4] = 128                # one flat frame
    a, b = proc(), proc()
    fa, oa = run_clip(a, fr[:5], cfg)
    fb, ob = run_frames(b, fr[:5], cfg)
    assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
    fa, oa = run_clip(a, fr[5:], cfg)
    fb, ob = run_frames(b, fr[5:], cfg)
    assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
    assert_all_states_equal(a, b)
    a.close()
    b.close()


def test_phase_clip_gray_is_passthrough():
    got = check_clip(O.MODE_PHASE, PHASE_UI, 131, 75, 1, [("clip", 4), ("clip", 3)])
    assert not any(g.any() for g in got)


@pytest.mark.parametrize("pinned", [False, True])
def test_phase_clip_host_path_multi_lane(pinned):
    """mc_process_clip on a 3-lane handle with a held lane, pageable or pinned buffers, equals frame calls"""
    torch = pytest.importorskip("torch")
    if pinned and not torch.cuda.is_available():
        pytest.skip("pinned host buffers need a CUDA device")
    cfg, _ = make_cfgs(O.MODE_PHASE, *PHASE_UI)
    w, h, c, lanes = 131, 75, 3, 3
    a, b = proc(lanes), proc(lanes)
    t = 0
    for n in (3, 4):
        if t:
            a.hold_lane(1)
            b.hold_lane(1)
        fr = clip_frames(t, n, lanes, w, h, c)
        if pinned:
            pin_in = torch.from_numpy(fr).pin_memory()
            pin_out = torch.full(fr.shape, SENTINEL, dtype=torch.uint8).pin_memory()
            fa = np.zeros((n, lanes), np.uint8)
            prm = _to_mc(cfg)
            a._check(a._lib.mc_process_clip(a._h, pin_in.data_ptr(), n, w, h, c, w * c, C.byref(prm), pin_out.data_ptr(), w * c,
                                            fa.ctypes.data_as(U8P)))
            oa = pin_out.numpy()
        else:
            fa, oa = run_clip(a, fr, cfg)
        fb, ob = run_frames(b, fr, cfg)
        assert np.array_equal(fa, fb) and np.array_equal(oa, ob)
        t += n
    assert_all_states_equal(a, b, (0, 2))
    a.close()
    b.close()


def test_phase_clip_profile_names_the_kernel():
    cfg, _ = make_cfgs(O.MODE_PHASE, *phase_ui(4))
    p = proc(1, (("profile_kernels", 1),))
    run_clip(p, clip_frames(0, 3, 1, 131, 75, 3), cfg)
    prof = p.profile_read()
    for lvl in range(3):
        assert prof[("riesz_phase_clip", lvl)][0] == 1 and ("riesz_phase", lvl) not in prof
    p.close()


def check_launches_per_clip(w=83, h=45, levels=3):
    """on a continuing handle a T = 2 and a T = 16 clip each add the launches of one frame call: 4L - 2"""
    cfg, _ = make_cfgs(O.MODE_PHASE, *phase_ui(levels))
    p = proc()
    run_clip(p, clip_frames(0, 2, 1, w, h, 3), cfg)
    n0 = p.launch_count
    run_frames(p, clip_frames(2, 1, 1, w, h, 3), cfg)
    per_frame = p.launch_count - n0
    assert per_frame == 4 * levels - 2
    t = 3
    for n in (2, 16):
        n0 = p.launch_count
        run_clip(p, clip_frames(t, n, 1, w, h, 3), cfg)
        assert p.launch_count - n0 == per_frame, n
        t += n
    p.close()


def test_phase_clip_launch_count():
    check_launches_per_clip()
