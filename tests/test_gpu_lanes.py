"""Lane lifecycle of a multi-lane handle (mc_restart_lane / mc_hold_lane / mc_lane_produced): every lane must behave,
bit for bit, like its own 1-lane MagnificationProcessor fed the same frames — restarted where the lane is restarted,
not fed at all while the lane is held."""
import ctypes as C
import os

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs

LAPLACE_UI = (20, 50.0, 0.4, 3.0, 40, 4)
PHASE_UI = (50, 50.0, 0.4, 3.0, 0, 3)
COLOR_UI = (100, 0.0, 0.8, 1.2, 0, 2)
SENTINEL = 0xA5
PHASE_STATES = ("old.lowpass", "old.rx", "old.ry", "phase.c", "phase.s", "lo.r0.c", "lo.r1.s", "hi.r0.s", "hi.r1.c")


def proc(lanes=1, options=()):
    p = L.MagnificationProcessor(0, lanes=lanes)
    for k, v in options:
        p.set_option(k, v)
    return p


def lane_frame(t, k, w, h, c):
    return synth_frame(t, w, h, c, seed=101 * k)


def stack(t, lanes, w, h, c):
    return np.stack([lane_frame(t, k, w, h, c) for k in range(lanes)])


def process_raw(p, frames, cfg):
    """mc_process into a sentinel-filled buffer -> (produced, out, lane flags)."""
    out = np.full_like(frames, SENTINEL)
    hh, ww = frames.shape[1:3]
    c = 1 if frames.ndim == 3 else frames.shape[3]
    produced = p.process_host(frames.ctypes.data, ww, hh, c, ww * c, cfg, out.ctypes.data, ww * c)
    return produced, out, p.lane_produced()


def single_run(frames, cfg, options=()):
    """A 1-lane processor fed `frames` -> ([(produced, out)], processor)."""
    p = proc(1, options)
    return [p.process_image(f, cfg) for f in frames], p


def state_names(p, mode):
    if mode == O.MODE_PHASE:
        return [(n, l) for n in PHASE_STATES for l in range(8) if p.state_dims(n, l)[0]]
    return [(n, l) for n in ("lowpassHi", "lowpassLo") for l in range(8) if p.state_dims(n, l)[0]]


def assert_lane_state_equal(multi, lane, single, mode):
    names = state_names(single, mode)
    assert names
    for n, l in names:
        assert np.array_equal(multi.get_state(n, l)[lane], single.get_state(n, l)[0]), (n, l)


# ---------------------------------------------------------------------------------------------------------------------
# checks shared with the emulation suite (tests/test_emu_lanes.py)
# ---------------------------------------------------------------------------------------------------------------------
def check_restart(mode, ui, w, h, c, lanes=4, lane=2, at=3, n=6, options=()):
    """Restart `lane` before frame `at`: it equals a fresh processor started at `at`, the other lanes their uninterrupted
    processors, in outputs, per-lane flags and state planes."""
    cfg, _ = make_cfgs(mode, *ui)
    m = proc(lanes, options)
    got = []
    for t in range(n):
        if t == at:
            m.restart_lane(lane)
        produced, out, flags = process_raw(m, stack(t, lanes, w, h, c), cfg)
        got.append((produced, out, flags))
    for k in range(lanes):
        if k == lane:
            before, _ = single_run([lane_frame(t, k, w, h, c) for t in range(at)], cfg, options)
            after, sp = single_run([lane_frame(t, k, w, h, c) for t in range(at, n)], cfg, options)
            ref = before + after
        else:
            ref, sp = single_run([lane_frame(t, k, w, h, c) for t in range(n)], cfg, options)
        for t, ((sprod, sout), (_, out, flags)) in enumerate(zip(ref, got)):
            assert bool(flags[k]) == bool(sprod), (k, t)
            if sprod:
                assert np.array_equal(out[k], sout), (k, t)
            else:
                assert (out[k] == SENTINEL).all(), (k, t)
        assert_lane_state_equal(m, k, sp, mode)
    if mode == O.MODE_PHASE:   # the restarted lane passes through on its first frame while the others still produce
        assert list(got[at][2]) == [k != lane for k in range(lanes)]
    m.close()


def check_hold(mode, ui, w, h, c, lanes=4, lane=1, span=(2, 5), n=7, options=()):
    """Hold `lane` for frames span[0] .. span[1]-1: flags are 0 there and its bytes of `out` keep the sentinel, its state
    is untouched, and afterwards it equals a processor that never saw those frames."""
    cfg, _ = make_cfgs(mode, *ui)
    m = proc(lanes, options)
    got, kept = [], None
    for t in range(n):
        if t == span[0]:
            m.hold_lane(lane)
            kept = {k: m.get_state(*k)[lane].copy() for k in state_names(m, mode)}
        if t == span[1]:
            assert all(np.array_equal(m.get_state(*k)[lane], v) for k, v in kept.items())
            m.hold_lane(lane, False)
        got.append(process_raw(m, stack(t, lanes, w, h, c), cfg))
    for t in range(*span):
        assert list(got[t][2]) == [k != lane for k in range(lanes)], t
        assert (got[t][1][lane] == SENTINEL).all(), t
    ts = [t for t in range(n) if not span[0] <= t < span[1]]
    ref, _ = single_run([lane_frame(t, lane, w, h, c) for t in ts], cfg, options)
    for t, (sprod, sout) in zip(ts, ref):
        assert bool(got[t][2][lane]) == bool(sprod), t
        if sprod:
            assert np.array_equal(got[t][1][lane], sout), t
    m.close()


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("c", [3, 1])
@pytest.mark.parametrize("options,lanes", [((), 4), ((("lane_groups", 2),), 16), ((("faithful_level0", 1),), 4)])
def test_laplace_restart_lane(c, options, lanes):
    check_restart(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, c, lanes=lanes, options=options)


@pytest.mark.parametrize("options", [(), (("band_from_state", 0),), (("egress_strip", 0),)])
def test_laplace_restart_lane_other_paths(options):
    check_restart(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, options=options)


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_hold_lane(c):
    check_hold(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, c)


def test_laplace_hold_lane_with_lane_groups():
    check_hold(O.MODE_LAPLACE, LAPLACE_UI, 131, 75, 3, lanes=16, lane=9, options=(("lane_groups", 2),))


def test_laplace_hold_keeps_device_output():
    """mc_process_device: the held lane's bytes of d_out are not written."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("device buffers need a CUDA device")
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    w, h, c, lanes = 131, 75, 3, 4
    m = proc(lanes)
    for t in range(4):
        if t == 2:
            m.hold_lane(1)
        d_in = torch.from_numpy(stack(t, lanes, w, h, c)).cuda()
        d_out = torch.full_like(d_in, SENTINEL)
        torch.cuda.synchronize()
        assert m.process_device(d_in.data_ptr(), w, h, c, w * c, cfg, d_out.data_ptr(), w * c)
        m.sync()
        out = d_out.cpu().numpy()
        flags = m.lane_produced()
        if t >= 2:
            assert list(flags) == [True, False, True, True]
            assert (out[1] == SENTINEL).all()
        else:
            assert flags.all() and not (out[1] == SENTINEL).all()
    m.close()


def test_laplace_analysis_only_restart():
    """analysis_only: a restarted lane's first frame is produced (as the handle's first frame is), the others are not."""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    w, h, c, lanes = 131, 75, 3, 3
    m = proc(lanes, (("analysis_only", 1),))
    single = proc(1, (("analysis_only", 1),))
    for t in range(3):
        process_raw(m, stack(t, lanes, w, h, c), cfg)
    m.restart_lane(1)
    produced, out, flags = process_raw(m, stack(3, lanes, w, h, c), cfg)
    sprod, sout = single.process_image(lane_frame(3, 1, w, h, c), cfg)
    assert produced and sprod and list(flags) == [False, True, False]
    assert np.array_equal(out[1], sout)
    assert (out[0] == SENTINEL).all() and (out[2] == SENTINEL).all()
    assert_lane_state_equal(m, 1, single, O.MODE_LAPLACE)


def test_phase_restart_lane():
    check_restart(O.MODE_PHASE, PHASE_UI, 120, 90, 3)


def test_phase_hold_lane():
    check_hold(O.MODE_PHASE, PHASE_UI, 120, 90, 3)


def test_phase_cutoff_change_while_held_restarts_the_lane():
    cfg, _ = make_cfgs(O.MODE_PHASE, *PHASE_UI)
    cfg2, _ = make_cfgs(O.MODE_PHASE, 50, 50.0, 0.6, 3.0, 0, 3)
    w, h, c, lanes, n = 120, 90, 3, 3, 7
    cfgs = [cfg if t < 3 else cfg2 for t in range(n)]
    m = proc(lanes)
    got = []
    for t in range(n):
        if t == 2:
            m.hold_lane(1)
        if t == 4:
            m.hold_lane(1, False)
        got.append(process_raw(m, stack(t, lanes, w, h, c), cfgs[t]))
    # the held lane: its first frame after release passes through, then it equals a fresh processor started there
    assert list(got[4][2]) == [True, False, True]
    fresh = proc(1)
    for t in range(4, n):
        sprod, sout = fresh.process_image(lane_frame(t, 1, w, h, c), cfgs[t])
        assert bool(got[t][2][1]) == bool(sprod), t
        if sprod:
            assert np.array_equal(got[t][1][1], sout), t
    # the running lanes go through the cutoff change as a single processor does
    for k in (0, 2):
        ref = proc(1)
        for t in range(n):
            sprod, sout = ref.process_image(lane_frame(t, k, w, h, c), cfgs[t])
            assert bool(got[t][2][k]) == bool(sprod), (k, t)
            if sprod:
                assert np.array_equal(got[t][1][k], sout), (k, t)


def test_hold_survives_structural_change_and_reset():
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    lanes = 4
    m = proc(lanes)
    size = lambda t: (131, 75) if t < 3 else (96, 64)
    got = []
    for t in range(7):
        if t == 2:
            m.hold_lane(1)
        if t == 5:
            m.hold_lane(1, False)
        w, h = size(t)
        got.append(process_raw(m, stack(t, lanes, w, h, 3), cfg))
    for k in range(lanes):
        start = 5 if k == 1 else 3   # the size change restarts every lane; the held one on release
        ref, _ = single_run([lane_frame(t, k, *size(t), 3) for t in range(start, 7)], cfg)
        for t, (sprod, sout) in zip(range(start, 7), ref):
            assert got[t][2][k] and np.array_equal(got[t][1][k], sout), (k, t)
    assert list(got[3][2]) == [True, False, True, True]
    # mc_reset: a pending restart is subsumed, holds stay
    m.restart_lane(2)
    m.hold_lane(3)
    m.reset()
    produced, out, flags = process_raw(m, stack(7, lanes, 96, 64, 3), cfg)
    assert list(flags) == [True, True, True, False] and (out[3] == SENTINEL).all()
    for k in range(3):
        sprod, sout = proc(1).process_image(lane_frame(7, k, 96, 64, 3), cfg)
        assert np.array_equal(out[k], sout), k


def check_pipelined(mode, ui, pinned, w, h):
    """Restarts and holds are taken at submit time: three frames in flight give the blocking path's frames and flags."""
    cfg, _ = make_cfgs(mode, *ui)
    c, lanes, n, depth = 3, 4, 9, 3
    events = {1: [("hold", 3, 1)], 2: [("restart", 0)], 4: [("hold", 3, 0), ("restart", 2)],
              5: [("restart", 1), ("hold", 2, 1)], 7: [("hold", 2, 0)]}

    def apply(p, t):
        for e in events.get(t, []):
            if e[0] == "hold":
                p.hold_lane(e[1], e[2])
            else:
                p.restart_lane(e[1])

    a, b = proc(lanes), proc(lanes)
    frames = [stack(t, lanes, w, h, c) for t in range(n)]
    ref = []
    for t in range(n):
        apply(a, t)
        ref.append(process_raw(a, frames[t], cfg))
    nbytes = frames[0].nbytes
    lib = capi.lib()
    if pinned:
        bufs = [lib.mc_host_alloc(nbytes) for _ in range(2 * n)]
        view = lambda p: np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=frames[0].shape)
        ins, outs = [view(p) for p in bufs[:n]], [view(p) for p in bufs[n:]]
        for t in range(n):
            ins[t][...] = frames[t]
    else:
        bufs, ins, outs = [], frames, [np.empty_like(frames[0]) for _ in range(n)]
    try:
        for o in outs:
            o[...] = SENTINEL
        got, done = [], 0
        for t in range(n):
            if t - done >= depth:
                got.append((b.collect(), b.lane_produced()))
                done += 1
            apply(b, t)
            b.submit(ins[t].ctypes.data, w, h, c, w * c, cfg, outs[t].ctypes.data, w * c)
        while done < n:
            got.append((b.collect(), b.lane_produced()))
            done += 1
        for t in range(n):
            assert got[t][0] == ref[t][0], t
            assert np.array_equal(got[t][1], ref[t][2]), t
            assert np.array_equal(outs[t], ref[t][1]), t
    finally:
        b.close()
        for p in bufs:
            lib.mc_host_free(p)


@pytest.mark.parametrize("mode,ui,pinned", [(O.MODE_LAPLACE, LAPLACE_UI, False), (O.MODE_LAPLACE, LAPLACE_UI, True),
                                            (O.MODE_PHASE, PHASE_UI, False)])
def test_pipelined_restarts_and_holds_equal_blocking(mode, ui, pinned):
    check_pipelined(mode, ui, pinned, 120, 90)


def test_color_multi_lane_refuses_and_keeps_its_window():
    cfg, _ = make_cfgs(O.MODE_COLOR, *COLOR_UI, 8.0)
    w, h, c, lanes, n = 90, 66, 3, 2, 14
    m, ref = proc(lanes), proc(lanes)
    frames = [stack(t, lanes, w, h, c) for t in range(n)]
    for t in range(n):
        if t == 5:   # a hold is refused while held; the window is as before
            m.hold_lane(1)
            with pytest.raises(L.MagcoreError) as e:
                m.process_image(frames[t], cfg)
            assert e.value.status == capi.MC_ERR_UNSUPPORTED
            m.hold_lane(1, False)
        if t == 9:   # a restart of one lane is refused until the handle is reset
            m.restart_lane(0)
            for _ in range(2):
                with pytest.raises(L.MagcoreError) as e:
                    m.process_image(frames[t], cfg)
                assert e.value.status == capi.MC_ERR_UNSUPPORTED
            m.reset()
            ref.close()
            ref = proc(lanes)
        p1, o1 = m.process_image(frames[t], cfg)
        p2, o2 = ref.process_image(frames[t], cfg)
        assert p1 == p2 and np.array_equal(o1, o2), t
        assert list(m.lane_produced()) == [p2] * lanes


def test_color_single_lane_restart_is_reset_and_hold_skips():
    cfg, _ = make_cfgs(O.MODE_COLOR, *COLOR_UI, 8.0)
    w, h, c, n = 90, 66, 3, 14
    frames = [lane_frame(t, 0, w, h, c) for t in range(n)]
    a, b = proc(1), proc(1)
    for t in range(n):
        if t == 6:
            a.restart_lane(0)
            b.reset()
        pa, oa = a.process_image(frames[t], cfg)
        pb, ob = b.process_image(frames[t], cfg)
        assert pa == pb and np.array_equal(oa, ob), t
    a, b = proc(1), proc(1)
    for t in range(n):
        if t in (6, 7):
            a.hold_lane(0)
            pa, oa = a.process_image(frames[t], cfg)
            assert not pa and oa is frames[t] and not a.lane_produced()[0]
            a.hold_lane(0, False)
            continue
        pa, oa = a.process_image(frames[t], cfg)
        pb, ob = b.process_image(frames[t], cfg)
        assert pa == pb and np.array_equal(oa, ob), t


def test_bad_lane_arguments():
    lib = capi.lib()
    m = proc(4)
    for call in (lambda: m.restart_lane(4), lambda: m.restart_lane(-1), lambda: m.hold_lane(4), lambda: m.hold_lane(-1)):
        with pytest.raises(L.MagcoreError) as e:
            call()
        assert e.value.status == capi.MC_ERR_INVALID
    buf = (C.c_uint8 * 8)()
    assert lib.mc_lane_produced(m._h, buf, 3) == capi.MC_ERR_INVALID
    assert lib.mc_lane_produced(m._h, buf, 5) == capi.MC_ERR_INVALID
    assert lib.mc_lane_produced(m._h, buf, 4) == capi.MC_OK
    chain = L.ProcessingChainB200(0)
    chain.magnifier.hold_lane(0)
    cfg, _ = make_cfgs(O.MODE_LAPLACE, *LAPLACE_UI)
    with pytest.raises(L.MagcoreError) as e:
        chain.run_chain_once(L.Frame(image=synth_frame(0, 64, 48, 3)), cfg)
    assert e.value.status == capi.MC_ERR_INVALID
    chain.magnifier.hold_lane(0, False)
    cur, _ = chain.run_chain_once(L.Frame(image=synth_frame(0, 64, 48, 3)), cfg)
    assert cur.image.shape == (48, 64, 3)


def test_process_image_fills_idle_lanes_with_their_input():
    cfg, _ = make_cfgs(O.MODE_PHASE, *PHASE_UI)
    m = proc(3)
    for t in range(3):
        if t == 2:
            m.restart_lane(0)
            m.hold_lane(2)
        f = stack(t, 3, 120, 90, 3)
        produced, out = m.process_image(f, cfg)
    assert produced and list(m.lane_produced()) == [False, True, False]
    assert np.array_equal(out[0], f[0]) and np.array_equal(out[2], f[2]) and not np.array_equal(out[1], f[1])


@pytest.mark.skipif(os.environ.get("MC_EMU") == "1", reason="full-HD frames are too slow for the CPU emulation")
def test_laplace_restart_and_hold_1080p():
    check_restart(O.MODE_LAPLACE, LAPLACE_UI, 1920, 1080, 3, lanes=2, lane=1, at=2, n=4)
    check_hold(O.MODE_LAPLACE, LAPLACE_UI, 1920, 1080, 3, lanes=2, lane=0, span=(1, 3), n=5)
