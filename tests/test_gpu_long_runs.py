"""Long free-running runs, every pipeline depth and the bench's own shape.

The stage tests isolate one kernel for one frame or one clip.  The checks here let the temporal state run free for as
long as a session runs, and run the configuration the headline number is measured on:

  content  pan_frame: a constant-velocity pan (0.7 or 1.3 px per frame, below and above a pixel per frame at the finest
           Phase level), a slow global brightness ramp for the EMA and the small oscillation of synth_frame, with seeded
           noise.  Its net motion drives the Phase integrator without bound, which synth_frame's oscillation never does.
  Phase    >= 2000 frames against the compiled reference (the oracle where it is absent): every frame <= 3 LSB and
           >= 99.5 % identical.  Every 250 frames phase.c / phase.s and the 8 DF-II registers against the oracle's
           RieszTemporalFilter, within a bound the run computes itself (PhaseBound), and |phase| must pass 300 rad.
  Laplace  >= 1500 frames at an EMA coefficient of 0.0104 (0.05 Hz at 30 fps), where the f32 update of a slowly moving
           plane is smaller than an ulp of the state: every frame <= 1 LSB, the state planes at checkpoints within
           test_gpu_laplace.run_pair's tolerance, and no drift: the largest relative state difference of the last window
           is no larger than that of the first window after the transient.
  Color    >= 600 frames cycling 8 / 15 / 30 / 60 fps (windows of 16, 32, 64, 128 frames), the changes landing right
           after a wrap, on a wrap, and on a partly filled ring: every frame <= 1 LSB, and after every frame the "window"
           tap is, column by column and bit for bit, the last n "gauss" taps, n the reference's window length.
  clips    the same runs fed to a second 2-lane handle as clips of 1, 7, 16, 33 and 64 frames, with a restart and a hold at
           clip boundaries: at each clip's end its outputs, flags and state planes (Color: every tap) equal the frame
           calls'.
  depth    pipeline_depth 1, 2, 5 and 16 over 200 frames of a 4-lane handle, BGR pageable and pinned for Laplace and
           Phase and mc_submit_nv12 for Laplace, with holds, a restart, a parameter change and a levels change while
           frames are in flight: the blocking calls' outputs, flags and state.  The option refuses 0, 17 and a change
           while frames are in flight.
  bench    64 lanes of 1920 x 1080 x 3, 6 levels, the bench's UI values and default options, lane k the base clip rolled
           as bench.make_clip rolls it, 40 steps of pinned submit / collect at depth 3: every lane equals a 1-lane handle
           fed that lane's frames in blocking calls, lanes 0 and 63 are within 1 LSB of the compiled reference for the
           first 8 steps; again with lane_groups 1.

The functions take their sizes and lengths as arguments; tests/test_emu_long_runs.py runs them on the CUDA-on-CPU
emulation at reduced sizes and lengths."""
import functools
import os
import time

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from oracle import livim_ref
from common import make_cfgs, planar, u8_diff
from test_gpu_clip import assert_states_equal, run_clip, run_frames
from test_gpu_lanes import SENTINEL, proc, process_raw
from test_gpu_nv12 import Dev, Layout, _pinned, to_nv12
from test_gpu_phase_clip import assert_all_states_equal

R = livim_ref.load()
if R is None and os.environ.get("MC_REQUIRE_REF") == "1":
    raise RuntimeError("MC_REQUIRE_REF=1 but oracle/_ref/_livim_ref is missing: run __graft_entry__.build() where "
                       "the reference sources are present, and keep oracle/_ref/ with the tree")
F32, F64 = np.float32, np.float64
LIFECYCLE = (("color_lane_lifecycle", 1),)
CLIP_LENGTHS = (1, 7, 16, 33, 64)
# (fps, frames): 8 fps (16) wraps at 16 and changes one frame after; 30 fps (64) changes on a ring filled to 36 of 64;
# 15 fps (32) shrinks it and wraps; 60 fps (128) grows and wraps; later changes land on a wrap (15 fps for 64 frames)
# and on partly filled rings again
COLOR_SCHEDULE = ((8.0, 17), (30.0, 20), (15.0, 40), (60.0, 150), (8.0, 33), (60.0, 97), (30.0, 65), (15.0, 64),
                  (8.0, 48), (30.0, 70))


# ---- content ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4096)
def pan_frame(t, w, h, vel, seed=0):
    """Frame t of a seeded clip with net motion: three oriented gratings (wavelengths 12, 24, 40 px) translating at `vel`
    px per frame along x (0.4 `vel` along y) plus synth_frame's 0.3 px oscillation at 1.5 Hz (30 fps), a global
    brightness ramp of 0.01 grey levels per frame, and +-2 LSB of noise from a generator seeded by (seed, t)."""
    yy, xx = np.mgrid[0:h, 0:w].astype(F64)
    s = vel * t + 0.3 * np.sin(2 * np.pi * 1.5 * t / 30.0)
    img = np.full((h, w, 3), 100.0 + 0.01 * t)
    for i, lam in enumerate((12, 24, 40)):
        th = i * np.pi / 5
        u = (xx + s) * np.cos(th) + (yy + 0.4 * s) * np.sin(th)
        for c in range(3):
            img[:, :, c] += 30.0 * np.sin(2 * np.pi * u / lam + 0.7 * c + 0.3 * i)
    img += np.random.default_rng([seed, t]).integers(-2, 3, size=(h, w, 3))
    out = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    out.setflags(write=False)
    return out


def lanes_frame(t, w, h, vel, lanes):
    """[lanes][h][w][3]: lane k is pan_frame rolled by 13 k px along x and carries its own noise"""
    return np.stack([np.roll(pan_frame(t, w, h, vel, seed=k), 13 * k, axis=1) for k in range(lanes)])


def eff_levels(w, h, levels):
    return min(max(levels, 1), O.calculate_max_levels(w, h))


class RefCore:
    """The compiled reference's magnification core (R.Core: magnifyMotion / magnifyColor / magnifyRiesz with their
    state structs) for one mode and a fixed geometry, or the oracle's where the compiled reference is absent."""

    def __init__(self, mode):
        self.mode = mode
        self.core = R.Core() if R is not None else None
        self.st = {O.MODE_LAPLACE: O.MotionState, O.MODE_PHASE: O.RieszState, O.MODE_COLOR: O.ColorState}[mode]()

    def run(self, frame, ocfg):
        p = ocfg.magnification
        h, w = frame.shape[:2]
        lv, c = eff_levels(w, h, p.levels), 1 if frame.ndim == 2 else frame.shape[2]
        if self.core is not None:
            return self.core.run(self.mode, frame, livim_ref.to_ref_params(R, p), lv)
        fn = {O.MODE_LAPLACE: O.magnify_motion, O.MODE_PHASE: O.magnify_riesz, O.MODE_COLOR: O.magnify_color}[self.mode]
        return fn(frame, p, lv, c, self.st)

    def motion_state(self):
        if self.core is not None:
            return self.core.motion_state()
        return self.st.lowpassHi, self.st.lowpassLo

    def window(self):
        return self.core.color_window() if self.core is not None else self.st.window


def check_phase_output(out, ref, where):
    d = u8_diff(out, ref)
    assert int(d.max()) <= 3 and float((d == 0).mean()) >= 0.995, (where, int(d.max()), float((d == 0).mean()))
    return int(d.max())


# ---- Phase -----------------------------------------------------------------------------------------------------------
def iir_gains(b, a, n):
    """DF-II of order 2 (y = b0 x + r0, r0' = b1 x + r1 - a1 y, r1' = b2 x - a2 y) in float64 over n frames ->
    (g_in, g_state): the largest sum over k < n of |register response| at lag k to a unit change of the input x, and
    to a unit change of one register (the infinity norm of the state transition's powers)."""
    A = np.array([[-a[1], 1.0], [-a[2], 0.0]])
    v = np.array([b[1] - a[1] * b[0], b[2] - a[2] * b[0]])
    M, g_in, g_state = np.eye(2), 0.0, 0.0
    for _ in range(n):
        g_in += float(np.abs(M @ v).max())
        g_state += float(np.abs(M).sum(axis=1).max())
        M = A @ M
    return g_in, g_state


class PhaseBound:
    """How far the device's phase integrator and DF-II registers may be from the oracle's after t frames, computed from
    the run itself.

    Every Phase operation of k_riesz_phase is correctly rounded and equals the reference's bit for bit (the stage tests
    of tests/test_gpu_phase_stages.py), except acosf, which CUDA bounds by 2 ulp where glibc's is within 1 ulp.  So on
    a frame the phase difference pd = o * acos(tmp) (|o| <= 1, o the direction qx / |q| or qy / |q|) can differ by
    2 ulp(acos) |o| <= 4 ulp(pd) (as x 2^-24 < ulp(x) <= x 2^-23), plus one ulp(pd) for the two products' roundings; the
    integrator's add of that frame rounds the two sums apart by at most one ulp of the integrator.  The integrator never
    forgets, so per pixel
        E_t = sum over frames s <= t of 5 ulp(|pd_s|) + ulp(|phase_s|).
    The registers are a linear function of the integrator's history plus their own roundings: with g_in and g_state of
    iir_gains over the run's length, a register may differ by
        g_in max E_t + g_state 16 ulp(m_t)
    where m_t bounds every intermediate of the plane so far (4 max |phase|: |b1|, |a1| <= 2) and 16 ulp covers the 9
    roundings of one DF-II step, each at most one ulp of its intermediate, carried through a1 and a2."""

    def __init__(self, oproc, levels, n):
        self.lv = levels
        self.E = [[0.0, 0.0] for _ in range(levels - 1)]
        self.m = [0.0] * (levels - 1)
        rz = oproc.riesz
        self.g = {f: iir_gains(filt.B, filt.A, n) for f, filt in (("lo", rz.lo), ("hi", rz.hi))}

    def add(self, oproc, debug):
        rz = oproc.riesz
        for lvl in range(self.lv - 1):
            for k in range(2):
                pd, ph = debug["phase_diff"][lvl][k], rz.lo.phase[lvl][k]
                self.E[lvl][k] = self.E[lvl][k] + 5 * np.spacing(np.abs(pd)).astype(F64) + np.spacing(np.abs(ph)).astype(F64)
                self.m[lvl] = max(self.m[lvl], 4.0 * float(np.abs(ph).max()))

    def registers(self, f, lvl):
        g_in, g_state = self.g[f]
        e = max(float(self.E[lvl][0].max()), float(self.E[lvl][1].max()))
        return g_in * e + g_state * 16 * float(np.spacing(F32(self.m[lvl])))


def phase_long_run(w, h, levels, n, vel, low=0.4, high=3.0, every=250, min_phase=300.0):
    """-> dict of what the run reached: the largest |phase|, and the largest observed difference / its bound of the
    integrator and the registers."""
    cfg, ocfg = make_cfgs(O.MODE_PHASE, 50, 50.0, low, high, 0, levels, 30.0)
    lv = eff_levels(w, h, levels)
    dev, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    ref = RefCore(O.MODE_PHASE) if R is not None else None
    bound, stats = None, {"phase": 0.0, "d_phase": 0.0, "d_phase_rel": 0.0, "d_reg": 0.0, "d_reg_rel": 0.0, "lsb": 0}
    for t in range(n):
        f = pan_frame(t, w, h, vel)
        produced, out = dev.process_image(f, cfg)
        dbg = {}
        oprod, oout = oproc.process(f, ocfg, dbg)
        if ref is not None:
            oprod, oout = ref.run(f, ocfg)
        assert produced == bool(oprod), t
        if not produced:
            bound = PhaseBound(oproc, lv, n)
            continue
        stats["lsb"] = max(stats["lsb"], check_phase_output(out, oout, t))
        bound.add(oproc, dbg)
        if (t + 1) % every and t != n - 1:
            continue
        rz = oproc.riesz
        for lvl in range(lv - 1):
            for k, cs in enumerate("cs"):
                got, want = dev.get_state(f"phase.{cs}", lvl)[0, 0], rz.lo.phase[lvl][k]
                d = np.abs(got.astype(F64) - want)
                assert (d <= bound.E[lvl][k]).all(), (t, lvl, cs, float(d.max()), float(bound.E[lvl][k].max()))
                stats["phase"] = max(stats["phase"], float(np.abs(want).max()))
                stats["d_phase"] = max(stats["d_phase"], float(d.max()))
                stats["d_phase_rel"] = max(stats["d_phase_rel"], float((d / bound.E[lvl][k]).max()))
                for fname in ("lo", "hi"):
                    filt = getattr(rz, fname)
                    for r, regs in (("r0", filt.reg0), ("r1", filt.reg1)):
                        got = dev.get_state(f"{fname}.{r}.{cs}", lvl)[0, 0]
                        dr = float(np.abs(got.astype(F64) - regs[lvl][k]).max())
                        br = bound.registers(fname, lvl)
                        assert dr <= br, (t, lvl, fname, r, cs, dr, br)
                        stats["d_reg"] = max(stats["d_reg"], dr)
                        stats["d_reg_rel"] = max(stats["d_reg_rel"], dr / br)
    assert stats["phase"] > min_phase, stats        # the regime of a real pan is reached
    dev.close()
    return stats


# ---- Laplace ---------------------------------------------------------------------------------------------------------
def laplace_long_run(w, h, levels, n, chroma, vel=0.7, low=0.05, every=50, transient=500, window=250):
    """-> (largest u8 difference, {checkpoint frame: largest relative state difference})"""
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, low, 3.0, chroma, levels, 30.0)
    assert ocfg.magnification.coLow <= 0.0105         # the EMA coefficient of the slow plane
    lv = eff_levels(w, h, levels)
    dev, ref = L.MagnificationProcessor(0), RefCore(O.MODE_LAPLACE)
    worst, rel = 0, {}
    for t in range(n):
        f = pan_frame(t, w, h, vel)
        produced, out = dev.process_image(f, cfg)
        rprod, rout = ref.run(f, ocfg)
        assert produced and rprod, t
        d = int(u8_diff(out, rout).max())
        assert d <= 1, (t, d)
        worst = max(worst, d)
        if (t + 1) % every:
            continue
        r = 0.0
        for name, planes in zip(("lowpassHi", "lowpassLo"), ref.motion_state()):
            for lvl in range(1, lv):
                got, want = dev.get_state(name, lvl)[0], planar(planes[lvl])
                dd = float(np.abs(got - want).max())
                rng = float(np.abs(want).max()) + 1e-6
                assert dd < 1e-3 and dd / rng < 2e-5, (t, name, lvl, dd, rng)     # test_gpu_laplace.run_pair
                r = max(r, dd / rng)
        rel[t + 1] = r
    first = max(v for k, v in rel.items() if transient < k <= transient + window)
    last = max(v for k, v in rel.items() if k > n - window)
    assert last <= first, (first, last, rel)
    dev.close()
    return worst, rel


# ---- Color -----------------------------------------------------------------------------------------------------------
def color_fps(t, schedule=COLOR_SCHEDULE):
    """the frame rate of frame t; the schedule repeats"""
    total = sum(k for _, k in schedule)
    t %= total
    for fps, k in schedule:
        if t < k:
            return fps
        t -= k


def color_long_run(w, h, n, levels=2, schedule=COLOR_SCHEDULE, lengths=(16, 32, 64, 128)):
    dev, ref = L.MagnificationProcessor(0), RefCore(O.MODE_COLOR)
    lv = eff_levels(w, h, levels)
    hist, worst, seen = [], 0, set()
    for t in range(n):
        fps = color_fps(t, schedule)
        cfg, ocfg = make_cfgs(O.MODE_COLOR, 100, 0.0, 0.8, 1.2, 0, levels, fps)
        f = pan_frame(t, w, h, 0.7)
        produced, out = dev.process_image(f, cfg)
        rprod, rout = ref.run(f, ocfg)
        assert produced == bool(rprod), t
        if produced:
            d = int(u8_diff(out, rout).max())
            assert d <= 1, (t, fps, d)
            worst = max(worst, d)
        k = ref.window().shape[1]
        seen.add(k)
        hist = (hist + [dev.get_state("gauss", lv)[0]])[-k:]
        assert dev.state_dims("window", k)[0] == 0 and dev.state_dims("window", k - 1)[0] > 0, (t, k)
        for j in range(k):
            assert np.array_equal(dev.get_state("window", j)[0], hist[j]), (t, fps, j, k)
    assert set(lengths) <= seen, seen
    dev.close()
    return worst


# ---- clips over the same runs ----------------------------------------------------------------------------------------
def color_taps(p):
    """every column of "window", "filtered" and every level of "gauss", "up" the handle serves"""
    out = {}
    for name in ("gauss", "window", "filtered", "up"):
        lvl = 0
        while p.state_dims(name, lvl)[0]:
            out[name, lvl] = p.get_state(name, lvl)
            lvl += 1
    return out


def long_clips(mode, w, h, n, levels, vel=1.3, lanes=2):
    """A 2-lane handle takes the run as clips of CLIP_LENGTHS (cycling), a twin the same frames as frame calls; lane 1
    restarts at every sixth clip boundary, lane 0 is held for every sixth clip.  Color changes its frame rate at clip
    starts (COLOR_SCHEDULE's rate of the clip's first frame) and runs with color_lane_lifecycle."""
    options = LIFECYCLE if mode == O.MODE_COLOR else ()
    a, b = proc(lanes, options), proc(lanes, options)
    t, i, clips_over_32 = 0, 0, 0
    while t < n:
        m = min(CLIP_LENGTHS[i % len(CLIP_LENGTHS)], n - t)
        fps = color_fps(t) if mode == O.MODE_COLOR else 30.0
        ui = {O.MODE_LAPLACE: (20, 50.0, 0.05, 3.0, 50, levels), O.MODE_PHASE: (50, 50.0, 0.4, 3.0, 0, levels),
              O.MODE_COLOR: (100, 0.0, 0.8, 1.2, 0, levels)}[mode]
        cfg, _ = make_cfgs(mode, *ui, fps)
        for p in (a, b):
            if i % 6 == 2:
                p.restart_lane(1)
            if i % 6 in (3, 4):
                p.hold_lane(0, i % 6 == 3)
        frames = np.stack([lanes_frame(s, w, h, vel, lanes) for s in range(t, t + m)])
        fa, oa = run_clip(a, frames, cfg)
        fb, ob = run_frames(b, frames, cfg)
        assert np.array_equal(fa, fb), (t, m)
        assert np.array_equal(oa, ob), (t, m)
        assert np.array_equal(a.lane_produced(), b.lane_produced()), (t, m)
        if mode == O.MODE_PHASE:
            assert_all_states_equal(a, b)
        elif mode == O.MODE_LAPLACE:
            assert_states_equal(a, b, mode)
        else:
            ta, tb = color_taps(a), color_taps(b)
            assert sorted(ta) == sorted(tb), (t, m)
            for key in tb:
                x, y = ta[key], tb[key]
                if key[0] == "gauss" and i % 6 == 3:     # the held lane's pyramid is that of whatever its input held
                    x, y = x[1:], y[1:]
                assert np.array_equal(x, y), (t, m, key)
        clips_over_32 += m > 32
        t += m
        i += 1
    assert clips_over_32 >= 2
    a.close()
    b.close()


# ---- pipeline depth --------------------------------------------------------------------------------------------------
DEPTH_KINDS = ("laplace-pageable", "laplace-pinned", "phase-pageable", "phase-pinned", "laplace-nv12",
               "laplace-nv12-pinned")


def depth_cfg(mode, t, n):
    """amplification 20 -> 35 at n/4 (no reset), Phase cutoffs 0.4 -> 0.6 Hz at n/2 (registers reset), levels 4 -> 3 at
    3n/5 (a structural reset of every lane)"""
    amp = (20 if mode == O.MODE_LAPLACE else 50) if t < n // 4 else 35
    low = 0.6 if mode == O.MODE_PHASE and t >= n // 2 else 0.4
    levels = 4 if t < 3 * n // 5 else 3
    return make_cfgs(mode, amp, 50.0, low, 3.0, 30 if mode == O.MODE_LAPLACE else 0, levels)[0]


def depth_events(n):
    """{frame: [event]} before that frame: two holds (one across the levels change), restarts of running and held lanes"""
    q = n // 20
    return {2 * q: [("hold", 3, 1)], 4 * q: [("hold", 3, 0), ("restart", 1)], 7 * q: [("restart", 2)],
            11 * q: [("hold", 0, 1)], 13 * q: [("restart", 0)], 15 * q: [("hold", 0, 0), ("hold", 2, 1)],
            16 * q: [("restart", 3)], 18 * q: [("hold", 2, 0)]}


def apply_events(p, events, t):
    for e in events.get(t, []):
        p.hold_lane(e[1], e[2]) if e[0] == "hold" else p.restart_lane(e[1])


def check_depth(kind, depth, w, h, n=200, lanes=4):
    """submit / collect with `depth` frames in flight equals the same calls made blocking: outputs (the sentinel where a
    lane did not produce), per-lane flags and every state plane afterwards."""
    mode = O.MODE_PHASE if kind.startswith("phase") else O.MODE_LAPLACE
    nv12, pinned = "nv12" in kind, kind.endswith("pinned")
    lib = capi.lib()
    events = depth_events(n)
    frames = [lanes_frame(t, w, h, 1.3, lanes) for t in range(n)]
    lay = Layout(w, h)
    if nv12:
        frames = [lay.pack(np.stack([to_nv12(f) for f in fr])) for fr in frames]
    a, b = proc(lanes), proc(lanes)
    # the option: 1 .. 16, and only while nothing is in flight
    for bad in (0, 17):
        assert lib.mc_set_option(b._h, b"pipeline_depth", bad) == capi.MC_ERR_INVALID
    assert lib.mc_pipeline_depth(b._h) == 3
    b.set_option("pipeline_depth", depth)
    assert lib.mc_pipeline_depth(b._h) == depth
    ref = []
    for t in range(n):
        apply_events(a, events, t)
        cfg = depth_cfg(mode, t, n)
        if nv12:
            d_in, d_out = Dev(frames[t]), Dev(np.full_like(frames[t], SENTINEL))
            prod = a.process_nv12_device(lay.planes(d_in.ptr), w, h, cfg, lay.planes(d_out.ptr))
            a.sync()
            ref.append((prod, a.lane_produced(), d_out.numpy()))
        else:
            prod, out, flags = process_raw(a, frames[t], cfg)
            ref.append((prod, flags, out))
    keep = []
    try:
        if pinned:
            ins = _pinned(lib, (n,) + frames[0].shape, keep)
            outs = _pinned(lib, (n,) + frames[0].shape, keep)
            ins[...] = np.stack(frames)
        else:
            ins, outs = np.stack(frames), np.empty((n,) + frames[0].shape, np.uint8)
        outs[...] = SENTINEL
        got, done = [], 0
        for t in range(n):
            if t - done >= depth:
                got.append((b.collect(), b.lane_produced()))
                done += 1
            apply_events(b, events, t)
            cfg = depth_cfg(mode, t, n)
            if nv12:
                b.submit_nv12(lay.planes(ins[t].ctypes.data), w, h, cfg, lay.planes(outs[t].ctypes.data))
            else:
                b.submit(ins[t].ctypes.data, w, h, 3, w * 3, cfg, outs[t].ctypes.data, w * 3)
            if t == n // 3:      # frames in flight: the depth stays
                assert lib.mc_set_option(b._h, b"pipeline_depth", 1 + depth % 16) == capi.MC_ERR_INVALID
                assert lib.mc_pipeline_depth(b._h) == depth
        while done < n:
            got.append((b.collect(), b.lane_produced()))
            done += 1
        for t in range(n):
            assert got[t][0] == ref[t][0], t
            assert np.array_equal(got[t][1], ref[t][1]), t
            assert np.array_equal(outs[t], ref[t][2]), t
        if mode == O.MODE_PHASE:
            assert_all_states_equal(b, a)
        else:
            assert_states_equal(b, a, mode)
        assert not all(r[1].all() for r in ref) and any(r[1].all() for r in ref)
    finally:
        b.close()
        for p in keep:
            lib.mc_host_free(p)


# ---- the bench's shape -----------------------------------------------------------------------------------------------
BENCH_UI = (20, 50.0, 0.4, 3.0, 0, 6)      # bench.UI: alpha 20, 0.4 - 3 Hz, chroma 0, 6 levels, 30 fps


def bench_shape(w, h, lanes, steps, clip_frames=8, ref_steps=8, ref_lanes=None, groups=(None, 1)):
    """`lanes` lanes stepped through pinned mc_submit / mc_collect at depth 3, as bench.py's end-to-end loop does, on one
    handle per entry of `groups` (None: the default lane_groups).  Every lane of every handle equals a 1-lane handle fed
    that lane's frames in blocking calls, stepped in lock-step with the collects; `ref_lanes` are checked against the
    compiled reference for the first `ref_steps` steps."""
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, *BENCH_UI, 30.0)
    c, depth, lib = 3, 3, capi.lib()
    ref_lanes = (0, lanes - 1) if ref_lanes is None else ref_lanes
    base = [synth_frame(t, w, h, c) for t in range(clip_frames)]
    multis = []
    for g in groups:
        m = L.MagnificationProcessor(0, lanes=lanes)
        if g is not None:
            m.set_option("lane_groups", g)
        multis.append(m)
    singles = [L.MagnificationProcessor(0) for _ in range(lanes)]
    refs = {k: RefCore(O.MODE_LAPLACE) for k in ref_lanes}
    keep = []
    shape = (lanes, h, w, c)
    try:
        ins = [_pinned(lib, shape, keep) for _ in range(depth)]
        outs = [[_pinned(lib, shape, keep) for _ in range(depth)] for _ in multis]
        single_out = np.empty((h, w, c), np.uint8)
        worst = 0

        def check(s):
            nonlocal worst
            slot = s % depth
            flags = []
            for m in multis:
                assert m.collect()
                flags.append(m.lane_produced())
            for k in range(lanes):
                f = ins[slot][k]
                assert singles[k].process_host(f.ctypes.data, w, h, c, w * c, cfg, single_out.ctypes.data, w * c)
                for g, (fl, o) in enumerate(zip(flags, outs)):
                    assert fl[k], (groups[g], s, k)
                    assert np.array_equal(o[slot][k], single_out), (groups[g], s, k)
                if s < ref_steps and k in refs:
                    rprod, rout = refs[k].run(np.ascontiguousarray(f), ocfg)
                    assert rprod
                    d = int(u8_diff(single_out, rout).max())
                    assert d <= 1, (s, k, d)
                    worst = max(worst, d)

        done = 0
        for s in range(steps):
            if s - done >= depth:
                check(done)
                done += 1
            slot = s % depth                           # collected: safe to refill
            for k in range(lanes):
                ins[slot][k] = np.roll(base[s % clip_frames], (11 * k, 37 * k), axis=(0, 1))
            for m, o in zip(multis, outs):
                m.submit(ins[slot].ctypes.data, w, h, c, w * c, cfg, o[slot].ctypes.data, w * c)
        while done < steps:
            check(done)
            done += 1
        for m in multis:
            for lvl in range(1, eff_levels(w, h, BENCH_UI[5])):
                for name in ("lowpassHi", "lowpassLo"):
                    st = m.get_state(name, lvl)
                    for k in (0, lanes // 2, lanes - 1):
                        assert np.array_equal(st[k], singles[k].get_state(name, lvl)[0]), (lvl, name, k)
        return worst
    finally:
        for m in multis + singles:
            m.close()
        for p in keep:
            lib.mc_host_free(p)


# ---------------------------------------------------------------------------------------------------------------------
pytestmark = pytest.mark.gpu
W, H = 96, 64


@pytest.mark.parametrize("vel,low,high", [(0.7, 0.4, 3.0), (1.3, 0.4, 3.0), (1.3, 0.02, 3.0), (1.3, 0.4, 15.0)],
                         ids=["pan0.7", "pan1.3", "low0.02Hz", "high_nyquist"])
def test_phase_long_run(vel, low, high):
    """2000 frames, 3 levels: every frame within the Phase tolerances of the reference, the integrator and registers
    within PhaseBound of the oracle every 250 frames.  0.02 Hz puts the low filter's poles at 0.994 and 15 Hz (Nyquist
    at 30 fps) the high filter's at -0.99999999, next to the unit circle."""
    t0 = time.time()
    s = phase_long_run(W, H, 3, 2000, vel, low, high)
    print(f"phase pan {vel} px/frame {low}-{high} Hz: max |phase| {s['phase']:.1f} rad, max |d phase| {s['d_phase']:.3g} "
          f"({s['d_phase_rel']:.3g} of its bound), max |d register| {s['d_reg']:.3g} ({s['d_reg_rel']:.3g} of its bound), "
          f"max u8 diff {s['lsb']}, {time.time() - t0:.1f} s")


@pytest.mark.parametrize("chroma", [0, 50])
def test_laplace_long_run(chroma):
    worst, rel = laplace_long_run(W, H, 4, 1500, chroma)
    print(f"laplace chroma {chroma}: max u8 diff {worst}, relative state difference per checkpoint "
          f"{ {k: f'{v:.2g}' for k, v in rel.items() if k % 250 == 0} }")


def test_color_long_run():
    worst = color_long_run(64, 48, sum(k for _, k in COLOR_SCHEDULE))
    print(f"color: max u8 diff {worst}")


@pytest.mark.parametrize("mode,n,levels", [(O.MODE_LAPLACE, 1500, 4), (O.MODE_PHASE, 2000, 3),
                                           (O.MODE_COLOR, sum(k for _, k in COLOR_SCHEDULE), 2)],
                         ids=["laplace", "phase", "color"])
def test_long_clips_equal_frame_calls(mode, n, levels):
    long_clips(mode, W, H, n, levels)


@pytest.mark.parametrize("kind", DEPTH_KINDS)
@pytest.mark.parametrize("depth", [1, 2, 5, 16])
def test_every_pipeline_depth_equals_blocking(kind, depth):
    check_depth(kind, depth, W, H)


def test_bench_shape_64_lanes_1080p():
    t0 = time.time()
    worst = bench_shape(1920, 1080, 64, 40)
    print(f"bench shape: 64 lanes 1920x1080, 40 steps at depth 3, lane_groups default and 1: max u8 diff of lanes 0, 63 "
          f"vs the reference {worst}, {time.time() - t0:.1f} s")
