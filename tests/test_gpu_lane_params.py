"""Per-lane parameters of a multi-lane handle (mc_set_lane_params): lane k, with the call's params where its override
replaces the six non-structural fields, must equal, bit for bit, a 1-lane handle fed lane k's frames with those params —
outputs, produced flags and the temporal state — under restarts, holds, and overrides set, changed and cleared mid-run,
through frame calls, clips and pipelined submits, in all three modes."""
import dataclasses

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from test_gpu_lanes import LAPLACE_UI, PHASE_UI, COLOR_UI, SENTINEL, lane_frame, process_raw, state_names

pytestmark = pytest.mark.gpu

FIELDS = ("amplification", "coWavelength", "coLow", "coHigh", "chromAttenuation", "framerate")


def mag(mode, ui, fps=30.0):
    """UI values (amplification, wavelength, low, high, chroma, levels) -> MagnificationParams, as the app forms them."""
    a, wl, lo, hi, ch, lv = ui
    return L.toParams(L.MagUiValues(mode=L.MagnificationMode(mode), amplification=a, wavelength=wl, low=lo, high=hi,
                                    chroma=ch, levels=lv, captureFps=fps))


def lane_ui(k, chroma=None):
    """A different Laplace UI per lane: gains, cutoffs, chroma and frame rate all vary."""
    return ((5 + 7 * k) % 41 + 1, 20.0 + (9 * k) % 61, 0.2 + 0.05 * (k % 8), 1.5 + 0.25 * (k % 9),
            [0, 50, 20, 100][k % 4] if chroma is None else chroma, 4), [25.0, 30.0, 60.0, 15.0][k % 4]


def effective(base, over):
    """The call's params with the six fields of `over` (None: the call's)."""
    return base if over is None else dataclasses.replace(base, **{f: getattr(over, f) for f in FIELDS})


def cfg_of(m):
    return L.ProcessorConfig(magnification=m)


def proc(lanes=1, options=()):
    p = L.MagnificationProcessor(0, lanes=lanes)
    for k, v in options:
        p.set_option(k, v)
    return p


# ---------------------------------------------------------------------------------------------------------------------
# checks shared with the emulation suite (tests/test_emu_lane_params.py)
# ---------------------------------------------------------------------------------------------------------------------
def check_lanes(mode, base_ui, w, h, c, overrides, n=6, schedule=None, options=(), entry="frame", clip=1, depth=3):
    """A `lanes`-lane handle with `overrides` (per lane: MagnificationParams or None) against one 1-lane twin per lane.
    schedule: {t: [("set", k, params|None) | ("restart", k) | ("hold", k, bool)]}, applied before frame t (for clips, t
    must be a multiple of `clip`; for submits the actions land while earlier frames are in flight).
    entry: "frame" (mc_process), "clip" (mc_process_clip of `clip` frames) or "submit" (pageable mc_submit at `depth`)."""
    lanes = len(overrides)
    schedule = schedule or {}
    base = mag(mode, base_ui)
    m = proc(lanes, options + ((("pipeline_depth", depth),) if entry == "submit" else ()))
    over = list(overrides)
    held = [False] * lanes
    for k, o in enumerate(over):
        if o is not None:
            m.set_lane_params(k, o)
    ins = [np.stack([lane_frame(t, k, w, h, c) for k in range(lanes)]) for t in range(n)]
    # the twins' view of every frame: (fed?, effective params)
    plan = []
    for t in range(n):
        for act in schedule.get(t, ()):
            if act[0] == "set":
                over[act[1]] = act[2]
            elif act[0] == "hold":
                held[act[1]] = act[2]
        plan.append(([not hd for hd in held], [effective(base, o) for o in over]))
    # ("twin_restart", k): only the twin restarts (the handle dropped the lane's state itself: a held lane's cutoff change)
    restarts = {t: [a[1] for a in acts if a[0] in ("restart", "twin_restart")] for t, acts in schedule.items()}

    def apply(t):
        for act in schedule.get(t, ()):
            if act[0] == "set":
                m.set_lane_params(act[1], act[2])
            elif act[0] == "restart":
                m.restart_lane(act[1])
            elif act[0] == "hold":
                m.hold_lane(act[1], act[2])

    got = []   # per frame: (flags, out)
    if entry == "frame":
        for t in range(n):
            apply(t)
            _, out, flags = process_raw(m, ins[t], cfg_of(base))
            got.append((flags.astype(bool), out))
    elif entry == "clip":
        assert n % clip == 0
        for t0 in range(0, n, clip):
            assert all(t not in schedule for t in range(t0 + 1, t0 + clip))
            apply(t0)
            flags, out = m.process_clip(np.stack(ins[t0:t0 + clip]), cfg_of(base))
            got += [(flags[i], out[i]) for i in range(clip)]
    else:
        outs = [np.full_like(ins[0], SENTINEL) for _ in range(n)]
        done = 0
        for t in range(n):
            if t - done >= depth:
                m.collect()
                got.append((m.lane_produced().astype(bool), outs[done]))
                done += 1
            apply(t)
            m.submit(ins[t].ctypes.data, w, h, c, w * c, cfg_of(base), outs[t].ctypes.data, w * c)
        while done < n:
            m.collect()
            got.append((m.lane_produced().astype(bool), outs[done]))
            done += 1
    for k in range(lanes):
        tw = proc(1, options)
        for t in range(n):
            if k in restarts.get(t, ()):
                tw.reset()
            fed, eff = plan[t]
            if not fed[k]:
                assert not got[t][0][k], (t, k)
                continue
            prod, out = tw.process_image(ins[t][k], cfg_of(eff[k]))
            assert bool(got[t][0][k]) == bool(prod), (entry, t, k)
            if prod:
                assert np.array_equal(got[t][1][k], out), (entry, t, k)
        for name, lv in state_names(tw, mode):
            assert np.array_equal(m.get_state(name, lv)[k], tw.get_state(name, lv)[0], equal_nan=True), (entry, k, name, lv)
    return m


def laplace_overrides(lanes, chroma=None, skip=()):
    base = mag(O.MODE_LAPLACE, LAPLACE_UI)
    out = []
    for k in range(lanes):
        ui, fps = lane_ui(k, chroma)
        out.append(None if k in skip else effective(base, mag(O.MODE_LAPLACE, ui, fps)))
    return out


def check_laplace_matrix(w, h):
    """Gray and colour, mixed chroma (L-only synthesis off) and all-zero chroma (on), both egress kernels, one and two
    lane groups, and the state-carry pass."""
    for c in (3, 1):
        check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, c, laplace_overrides(4, skip=(2,)))
    check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, laplace_overrides(4, chroma=0))
    check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, laplace_overrides(4), options=(("egress_strip", 0),))
    check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, laplace_overrides(4, chroma=0), options=(("egress_strip", 0),))
    for g in (1, 2):
        check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, laplace_overrides(4), options=(("lane_groups", g),))
    check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, laplace_overrides(3), options=(("analysis_only", 1),))


def check_schedule(w, h, entry="frame", clip=1, depth=3):
    """Overrides set, changed and cleared mid-run with a restart and a hold."""
    o = laplace_overrides(6)
    sched = {clip: [("set", 0, o[1]), ("hold", 3, True)], 2 * clip: [("set", 1, None), ("restart", 2)],
             3 * clip: [("hold", 3, False), ("set", 3, o[0])], 4 * clip: [("set", 2, o[5])]}
    check_lanes(O.MODE_LAPLACE, LAPLACE_UI, w, h, 3, [o[0], o[1], None, o[3]], n=5 * clip, schedule=sched, entry=entry,
                clip=clip, depth=depth)


def check_equal_override_is_none(w, h):
    """An override equal to the call's params gives the bytes and the launch count of no override."""
    lanes, base = 3, mag(O.MODE_LAPLACE, LAPLACE_UI)
    a, b = proc(lanes), proc(lanes)
    for k in range(lanes):
        b.set_lane_params(k, base)
    for t in range(4):
        f = np.stack([lane_frame(t, k, w, h, 3) for k in range(lanes)])
        ra, rb = process_raw(a, f, cfg_of(base)), process_raw(b, f, cfg_of(base))
        assert np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2])
    assert a.launch_count == b.launch_count


def phase_overrides():
    """Distinct cutoffs, amplifications, wavelengths and frame rates."""
    base = mag(O.MODE_PHASE, PHASE_UI)
    return [None] + [effective(base, mag(O.MODE_PHASE, ui, fps)) for ui, fps in
                     (((30, 40.0, 0.3, 2.0, 0, 3), 15.0), ((80, 70.0, 0.8, 4.5, 0, 3), 60.0))]


def check_phase(w, h, entry="frame", clip=1):
    """Phase lanes with their own filters; a cutoff change on one running lane (the others' state stays equal to their
    twins'), a cutoff change on a held lane (it restarts on release, as its twin after a reset), and a lane whose design
    is not finite (every frame of it is a first frame)."""
    o = phase_overrides()
    base = mag(O.MODE_PHASE, PHASE_UI)
    moved = dataclasses.replace(o[1], coLow=0.5, coHigh=2.5)
    nan = dataclasses.replace(base, coHigh=float("nan"))
    check_lanes(O.MODE_PHASE, PHASE_UI, w, h, 3, o, n=4 * clip, entry=entry, clip=clip)
    sched = {clip: [("hold", 2, True)], 2 * clip: [("set", 1, moved), ("set", 2, dataclasses.replace(o[2], coLow=0.6))],
             3 * clip: [("hold", 2, False), ("twin_restart", 2)]}
    check_lanes(O.MODE_PHASE, PHASE_UI, w, h, 3, o, n=5 * clip, schedule=sched, entry=entry, clip=clip)
    check_lanes(O.MODE_PHASE, PHASE_UI, w, h, 3, [o[1], nan, o[2]], n=3 * clip, entry=entry, clip=clip)


def check_color(w, h, n=40):
    """Color lanes at 8 / 15 / 30 fps (windows 16 / 32 / 64) with option color_lane_lifecycle: the windows fill, wrap,
    and change when a lane's rate changes mid-run."""
    base = mag(O.MODE_COLOR, COLOR_UI)
    o = [effective(base, mag(O.MODE_COLOR, COLOR_UI, fps)) for fps in (8.0, 15.0, 30.0)]
    o[1] = dataclasses.replace(o[1], amplification=60.0, coLow=0.6, coHigh=1.8)
    sched = {n // 2: [("set", 0, effective(base, mag(O.MODE_COLOR, COLOR_UI, 15.0)))]}
    check_lanes(O.MODE_COLOR, COLOR_UI, w, h, 3, o, n=n, schedule=sched, options=(("color_lane_lifecycle", 1),))


def check_color_refusal(w, h):
    """Without color_lane_lifecycle, Color lanes whose params differ are refused: the refused call changes nothing, so
    the handle goes on exactly as a handle that never saw it."""
    ui = COLOR_UI
    base = mag(O.MODE_COLOR, ui)
    a, b = proc(3), proc(3)
    frames = [np.stack([lane_frame(t, k, w, h, 3) for k in range(3)]) for t in range(6)]
    for t in range(3):
        ra, rb = process_raw(a, frames[t], cfg_of(base)), process_raw(b, frames[t], cfg_of(base))
    a.set_lane_params(1, effective(base, mag(O.MODE_COLOR, ui, 15.0)))
    with pytest.raises(capi.MagcoreError) as e:
        process_raw(a, frames[3], cfg_of(base))
    assert e.value.status == capi.MC_ERR_UNSUPPORTED
    a.set_lane_params(1, None)
    for t in range(3, 6):
        ra, rb = process_raw(a, frames[t], cfg_of(base)), process_raw(b, frames[t], cfg_of(base))
        assert np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2]), t


def check_errors():
    lib = capi.lib()
    m = proc(2)
    lp = capi.McLaneParams(1, 2, 0.1, 0.2, 0, 30)
    for bad in (-1, 2):
        assert lib.mc_set_lane_params(m._h, bad, lp) == capi.MC_ERR_INVALID
    assert lib.mc_set_lane_params(None, 0, lp) == capi.MC_ERR_INVALID
    assert lib.mc_set_lane_params(m._h, 1, None) == capi.MC_OK


# ---------------------------------------------------------------------------------------------------------------------
def test_laplace_lanes_with_their_own_params():
    check_laplace_matrix(166, 94)


@pytest.mark.parametrize("entry,clip,depth", [("frame", 1, 3), ("clip", 1, 3), ("clip", 7, 3), ("clip", 16, 3),
                                              ("submit", 1, 1), ("submit", 1, 3), ("submit", 1, 5)])
def test_schedules_on_every_entry_point(entry, clip, depth):
    check_schedule(166, 94, entry, clip, depth)


def test_override_equal_to_call_params_changes_nothing():
    check_equal_override_is_none(166, 94)


@pytest.mark.parametrize("entry,clip", [("frame", 1), ("clip", 7)])
def test_phase_lanes_with_their_own_params(entry, clip):
    check_phase(96, 64, entry, clip)


def test_color_lanes_with_their_own_rates():
    check_color(96, 64, n=80)


def test_color_refuses_different_params_without_lane_lifecycle():
    check_color_refusal(96, 64)


def test_errors():
    check_errors()


def test_bench_shape_64_lanes_1080p():
    """64 lanes of 1080p, 6 levels, 64 different params: every lane equals its 1-lane twin; lanes 0 and 63 are within
    1 LSB of the compiled reference run with their params."""
    from test_gpu_long_runs import RefCore, u8_diff
    w, h, c, lanes, n = 1920, 1080, 3, 64, 4
    base_ui = (20, 50.0, 0.4, 3.0, 0, 6)
    base = mag(O.MODE_LAPLACE, base_ui)
    uis = [lane_ui(k) for k in range(lanes)]
    over = [effective(base, mag(O.MODE_LAPLACE, ui, fps)) for ui, fps in uis]
    m = proc(lanes)
    for k, o in enumerate(over):
        m.set_lane_params(k, o)
    frames = [np.stack([np.roll(synth_frame(t, w, h, c), (11 * k, 37 * k), axis=(0, 1)) for k in range(lanes)]) for t in range(n)]
    outs = []
    for t in range(n):
        _, out, flags = process_raw(m, frames[t], cfg_of(base))
        assert flags.all()
        outs.append(out)
    for k in range(lanes):
        tw = proc(1)
        ref = RefCore(O.MODE_LAPLACE) if k in (0, lanes - 1) else None
        a, wl, lo, hi, ch, _ = uis[k][0]
        ocfg = O.ProcessorConfig(magnification=O.to_params(O.MODE_LAPLACE, a, wl, lo, hi, ch, 6, uis[k][1]))
        for t in range(n):
            prod, out = tw.process_image(frames[t][k], cfg_of(over[k]))
            assert prod and np.array_equal(outs[t][k], out), (t, k)
            if ref is not None:
                rprod, rout = ref.run(np.ascontiguousarray(frames[t][k]), ocfg)
                assert rprod and int(u8_diff(out, rout).max()) <= 1, (t, k)
