"""Motion (Laplace) parity: CUDA path (through the C ABI) vs the oracle, on an H100.

Tolerances (SURVEY.md §A.7 / BASELINE.md §3): f32 output in [0,1] units before 8-bit quantisation
max-abs < 1e-4; u8 output <= 1 LSB; state planes (Lab scale, L in [0,100]) max-abs < 1e-3 absolute
and < 1e-5 relative to the plane's dynamic range."""
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs, planar, u8_diff

pytestmark = pytest.mark.gpu

F32_TOL = 1e-4


def run_pair(w, h, c, levels, n, chroma=0, faithful=True, amplification=20, check_state=True):
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, amplification, 50.0, 0.4, 3.0, chroma, levels)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    proc.set_option("faithful_level0", int(faithful))
    proc.set_option("keep_float_output", 1)
    worst_f, worst_u8 = 0.0, 0
    for t in range(n):
        f = synth_frame(t, w, h, c)
        dbg = {}
        produced, out = proc.process_image(f, cfg)
        oprod, oout = oproc.process(f, ocfg, dbg)
        assert produced and oprod
        ref_f = dbg["output_bgr_f32"] if c == 3 else dbg["output_f32"]
        got_f = proc.float_output(w, h, c)[0]
        if c == 1:
            got_f = got_f[..., 0]
        worst_f = max(worst_f, float(np.abs(got_f - ref_f).max()))
        worst_u8 = max(worst_u8, int(u8_diff(out, oout).max()))
    lv_eff = min(max(levels, 1), L.calculateMaxLevels(w, h))
    if check_state:
        for name, ost in (("lowpassHi", oproc.motion.lowpassHi), ("lowpassLo", oproc.motion.lowpassLo)):
            for lvl in range(lv_eff + 1):
                got = proc.get_state(name, lvl)
                if got is None:
                    assert not faithful and lvl in (0, lv_eff)
                    continue
                ref = planar(ost[lvl])
                d = float(np.abs(got[0] - ref).max())
                rng = float(np.abs(ref).max()) + 1e-6
                assert d < 1e-3 and d / rng < 2e-5, (name, lvl, d, rng)
    return worst_f, worst_u8


@pytest.mark.parametrize("w,h,c,levels", [
    (320, 240, 3, 4), (320, 240, 1, 4), (240, 135, 3, 5), (135, 240, 1, 5), (67, 35, 3, 3), (30, 17, 1, 2),
    (64, 64, 3, 1), (7, 9, 3, 4), (130, 66, 3, 9),
])
def test_free_running_small(w, h, c, levels):
    wf, wu = run_pair(w, h, c, levels, 12, chroma=50)
    assert wf < F32_TOL, wf
    assert wu <= 1, wu


def test_config1_640x480():
    wf, wu = run_pair(640, 480, 3, 4, 32, chroma=0)
    assert wf < F32_TOL and wu <= 1, (wf, wu)


def test_config2_1080p_color_and_gray():
    for c in (3, 1):
        wf, wu = run_pair(1920, 1080, c, 6, 6, chroma=0)
        assert wf < F32_TOL and wu <= 1, (c, wf, wu)


def test_production_mode_matches_faithful():
    """Skipping the dead level-0 / residual state (default) must not change the output."""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, 5)
    a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
    a.set_option("faithful_level0", 1)
    for t in range(8):
        f = synth_frame(t, 322, 241, 3)
        _, oa = a.process_image(f, cfg)
        _, ob = b.process_image(f, cfg)
        assert np.array_equal(oa, ob)
    assert b.get_state("lowpassHi", 0) is None and b.get_state("lowpassHi", 1) is not None


def test_teacher_forced_single_step():
    """Inject the oracle's state for frame t-1, process frame t, compare output and new state."""
    w, h, c, levels = 322, 241, 3, 5
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 40, levels)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    proc.set_option("faithful_level0", 1)
    proc.set_option("keep_float_output", 1)
    for t in range(6):
        f = synth_frame(t, w, h, c)
        if t >= 1:
            for lvl in range(levels + 1):
                proc.set_state("lowpassHi", lvl, planar(oproc.motion.lowpassHi[lvl])[None])
                proc.set_state("lowpassLo", lvl, planar(oproc.motion.lowpassLo[lvl])[None])
        dbg = {}
        _, out = proc.process_image(f, cfg)
        _, oout = oproc.process(f, ocfg, dbg)
        assert float(np.abs(proc.float_output(w, h, c)[0] - dbg["output_bgr_f32"]).max()) < F32_TOL
        assert int(u8_diff(out, oout).max()) <= 1
        for lvl in range(levels):
            d = np.abs(proc.get_state("lowpassHi", lvl)[0] - planar(oproc.motion.lowpassHi[lvl])).max()
            assert d < 1e-3, (t, lvl, d)


def test_structural_reset_and_param_change():
    """levels / size / channel changes reset state (MagnifyCore.hpp:53-65); alpha/cutoff changes do not."""
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    seq = [(320, 240, 3, 4, 20, 0.4, 3.0)] * 4 + [(320, 240, 3, 4, 35, 0.8, 2.0)] * 3 + \
          [(320, 240, 3, 3, 35, 0.8, 2.0)] * 3 + [(200, 120, 1, 3, 35, 0.8, 2.0)] * 3
    for t, (w, h, c, lv, amp, lo, hi) in enumerate(seq):
        cfg, ocfg = make_cfgs(O.MODE_LAPLACE, amp, 50.0, lo, hi, 20, lv)
        f = synth_frame(t, w, h, c)
        produced, out = proc.process_image(f, cfg)
        oprod, oout = oproc.process(f, ocfg)
        assert produced == oprod and int(u8_diff(out, oout).max()) <= 1, t


def test_passthrough_and_reset_semantics():
    proc = L.MagnificationProcessor(0)
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 4)
    none_cfg = L.ProcessorConfig(magnification=L.MagnificationParams(mode=L.MagnificationMode.NONE))
    f = synth_frame(0, 64, 48, 3)
    fr = L.Frame(image=f, seq=7)
    assert proc.process(fr, none_cfg) is fr                      # mode None -> same FrameRef
    tiny = L.Frame(image=np.zeros((5, 40, 3), np.uint8))
    assert proc.process(tiny, cfg) is tiny                        # too small -> identity
    out = proc.process(fr, cfg)
    assert out is not fr and out.seq == 7 and out.image is not f  # fresh buffer, metadata kept
    # reset(): next frame behaves as the first frame again
    oproc = O.MagnificationProcessor()
    for t in range(3):
        proc.process_image(synth_frame(t, 64, 48, 3), cfg)
    proc.reset()
    _, o1 = proc.process_image(synth_frame(9, 64, 48, 3), cfg)
    _, r1 = oproc.process(synth_frame(9, 64, 48, 3), ocfg)
    assert int(u8_diff(o1, r1).max()) <= 1


def test_two_instances_and_lanes():
    """Instances are independent; a 3-lane handle equals three 1-lane handles bit for bit."""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 10, 4)
    singles = [L.MagnificationProcessor(0) for _ in range(3)]
    multi = L.MagnificationProcessor(0, lanes=3)
    for t in range(5):
        frames = [synth_frame(t, 160, 120, 3, seed=100 * k) for k in range(3)]
        outs = [p.process_image(f, cfg)[1] for p, f in zip(singles, frames)]
        _, mo = multi.process_image(np.stack(frames), cfg)
        for k in range(3):
            assert np.array_equal(mo[k], outs[k])


def test_pipelined_submit_collect_matches_blocking():
    import ctypes as C
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 4)
    a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
    w, h, c, n = 320, 240, 3, 9
    frames = [synth_frame(t, w, h, c) for t in range(n)]
    ref = [a.process_image(f, cfg)[1] for f in frames]
    outs = [np.empty_like(f) for f in frames]
    depth, done = 3, 0
    for t in range(n):
        if t - done >= depth:
            assert b.collect()
            done += 1
        b.submit(frames[t].ctypes.data, w, h, c, w * c, cfg, outs[t].ctypes.data, w * c)
    while done < n:
        assert b.collect()
        done += 1
    for t in range(n):
        assert np.array_equal(outs[t], ref[t]), t


def test_pipelined_submit_collect_with_pinned_buffers():
    """The zero-staging path of mc_submit: frames and results live in pinned memory (mc_host_alloc), so H2D / D2H go
    straight between the caller's buffers and HBM on the copy streams, three frames in flight, buffers reused round-robin
    as the bench's end-to-end loop does.  Same frames as the blocking API, for all three modes."""
    import ctypes as C
    from lvm_b200 import capi
    lib = capi.lib()
    w, h, c, depth = 320, 240, 3, 3
    nbytes = w * h * c
    for mode, ui, n in ((O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 4), 9), (O.MODE_PHASE, (50, 50.0, 0.4, 3.0, 0, 3), 7),
                        (O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 2), 7)):
        cfg, _ = make_cfgs(mode, *ui)
        a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
        frames = [synth_frame(t, w, h, c) for t in range(n)]
        ref = [a.process_image(f, cfg) for f in frames]
        ins = [lib.mc_host_alloc(nbytes) for _ in range(depth)]
        outs = [lib.mc_host_alloc(nbytes) for _ in range(depth)]
        assert all(ins) and all(outs)
        view = lambda p: np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(h, w, c))
        got, done = [], 0
        try:
            for t in range(n):
                if t - done >= depth:
                    produced = b.collect()
                    got.append(view(outs[done % depth]).copy() if produced else None)
                    done += 1
                view(ins[t % depth])[...] = frames[t]            # slot t % depth was collected: safe to refill
                b.submit(ins[t % depth], w, h, c, w * c, cfg, outs[t % depth], w * c)
            while done < n:
                produced = b.collect()
                got.append(view(outs[done % depth]).copy() if produced else None)
                done += 1
        finally:
            b.close()
            for p in ins + outs:
                lib.mc_host_free(p)
        for t, (g, (produced, r)) in enumerate(zip(got, ref)):
            assert (g is not None) == bool(produced), (mode, t)
            if produced:
                assert np.array_equal(g, r), (mode, t)


def test_cpp_adapter_runs_on_gpu():
    """The reference-side C++ IProcessor adapter (built against stub reference headers) magnifies a frame."""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "adapter_stub", "adapter_check")
    if not os.path.exists(exe):
        import __graft_entry__ as g
        g.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK gpu" in r.stdout, (r.returncode, r.stdout, r.stderr)


def test_tma_staging_equals_ldg_staging():
    """The fused level kernel stages its tiles with TMA (cp.async.bulk.tensor, zero-filled borders patched to
    REFLECT_101 in shared memory); option use_tma=0 selects the 128-bit LDG path.  Results must be identical,
    also for sizes whose border tiles are ragged."""
    for (w, h, c, lv) in [(640, 480, 3, 4), (333, 251, 1, 5), (1920, 1080, 3, 6)]:
        cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, lv)
        a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
        b.set_option("use_tma", 0)
        for t in range(4):
            f = synth_frame(t, w, h, c)
            _, oa = a.process_image(f, cfg)
            _, ob = b.process_image(f, cfg)
            assert np.array_equal(oa, ob), (w, h, t)
        for lvl in range(1, lv):
            assert np.array_equal(a.get_state("lowpassHi", lvl), b.get_state("lowpassHi", lvl))


def test_strided_rows_through_c_abi():
    """in_step / out_step larger than w*c (cv::Mat with padding, GL-style strides) — padding must be ignored
    on input and left untouched on output."""
    import ctypes as C
    from lvm_b200 import capi
    w, h, c, levels = 317, 203, 3, 4
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, levels)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    in_step, out_step = w * c + 13, w * c + 29
    lib = capi.lib()
    p = L.processor._to_mc(cfg)
    for t in range(4):
        f = synth_frame(t, w, h, c)
        src = np.full((h, in_step), 0xAB, np.uint8)
        src[:, :w * c] = f.reshape(h, w * c)
        dst = np.full((h, out_step), 0xCD, np.uint8)
        produced = C.c_int(0)
        st = lib.mc_process(proc._h, src.ctypes.data, w, h, c, in_step, C.byref(p), dst.ctypes.data, out_step, C.byref(produced))
        assert st == 0 and produced.value == 1
        _, ref = oproc.process(f, ocfg)
        assert int(u8_diff(dst[:, :w * c].reshape(h, w, c), ref).max()) <= 1
        assert (dst[:, w * c:] == 0xCD).all()


def test_levels_clamp_and_zero_amplification_properties():
    """levels above calculateMaxLevels are clamped (MagnificationProcessor.cpp:34); alpha = 0 makes every gain
    min(0, .) <= 0 ... = 0 only when the wavelength term is positive, so instead use the exact property that a
    static clip has a zero band-pass: output == the first-frame (Lab round-trip) output for every frame."""
    w, h, c = 322, 241, 3
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 50, 20)     # levels = 20 -> clamped to 6
    assert L.calculateMaxLevels(w, h) == 6
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    f = synth_frame(3, w, h, c)
    first = None
    for t in range(5):
        produced, out = proc.process_image(f, cfg)
        _, oout = oproc.process(f, ocfg)
        assert produced and int(u8_diff(out, oout).max()) <= 1
        if first is None:
            first = out
        else:
            assert np.array_equal(out, first), t      # identical frames -> hi == lo == band -> motion == 0 exactly
    assert proc.get_state("lowpassHi", 5) is not None and proc.get_state("lowpassHi", 6) is None


def test_config5_4k_8_levels():
    w, h, levels = 3840, 2160, 8
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, levels)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    proc.set_option("keep_float_output", 1)
    for t in range(3):
        f = synth_frame(t, w, h, 3)
        dbg = {}
        _, out = proc.process_image(f, cfg)
        _, oout = oproc.process(f, ocfg, dbg)
        assert float(np.abs(proc.float_output(w, h, 3)[0] - dbg["output_bgr_f32"]).max()) < F32_TOL
        assert int(u8_diff(out, oout).max()) <= 1


def test_empty_image_and_mode_none_free_state():
    proc = L.MagnificationProcessor(0)
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 4)
    proc.process_image(synth_frame(0, 64, 48, 3), cfg)
    assert proc.get_state("lowpassHi", 1) is not None
    produced, out = proc.process_image(np.zeros((0, 0, 3), np.uint8), cfg)        # empty image: identity, state dropped
    assert not produced
    assert proc.state_dims("lowpassHi", 1)[0] == 0
    produced, _ = proc.process_image(synth_frame(1, 64, 48, 3), cfg)              # starts again as a first frame
    assert produced


def test_band_from_state_option_equals_stored_band():
    """Option band_from_state (synthesis rebuilds gain*(hi-lo) from the state planes) must not change a single bit."""
    for (w, h, c, levels) in ((322, 241, 3, 5), (131, 75, 1, 3), (200, 120, 3, 2), (640, 360, 3, 6)):
        cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, levels)
        a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
        b.set_option("band_from_state", 0)
        for t in range(5):
            f = synth_frame(t, w, h, c)
            _, oa = a.process_image(f, cfg)
            _, ob = b.process_image(f, cfg)
            assert np.array_equal(oa, ob), (w, h, t)


@pytest.mark.parametrize("opts", [{"band_from_state": 0}, {"use_tma": 0}, {"egress_strip": 0}, {"egress_strip": 0, "band_from_state": 0},
                                  {"use_tma": 0, "band_from_state": 0}, {"use_tma": 0, "egress_strip": 0},
                                  {"use_tma": 0, "egress_strip": 0, "band_from_state": 0}, {"keep_float_output": 1}],
                         ids=lambda opts: ",".join(f"{k}={v}" for k, v in opts.items()))
def test_option_combinations_agree_with_default(opts):
    """The A/B options compose: every combination of band_from_state, use_tma and egress_strip, and the strip egress's
    float-tap instance, give the default path's frames bit for bit, over the first frame, ragged borders and a
    parameter change."""
    w, h, levels = 333, 251, 5
    a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
    for k, v in opts.items():
        b.set_option(k, v)
    for t in range(6):
        cfg, _ = make_cfgs(O.MODE_LAPLACE, 20 if t < 4 else 35, 50.0, 0.4, 3.0, 30, levels)
        f = synth_frame(t, w, h, 3)
        _, oa = a.process_image(f, cfg)
        _, ob = b.process_image(f, cfg)
        assert int(u8_diff(oa, ob).max()) == 0, (opts, t)


@pytest.mark.parametrize("w,h,c,lv", [(640, 480, 3, 4), (333, 251, 3, 5), (121, 75, 3, 3), (119, 64, 3, 3), (240, 67, 3, 2), (242, 130, 1, 3),
                                      (250, 131, 3, 2), (64, 48, 1, 2), (481, 270, 3, 6), (126, 129, 3, 3)])
def test_strip_egress_equals_tile_egress(w, h, c, lv):
    """The register/shuffle strip egress kernel (default) and the shared-memory tile kernel (option egress_strip = 0)
    collapse levels 2 -> 1 -> 0 with the same operations in the same order: bit-identical u8 frames and float taps,
    over ragged strips and chunks (widths around 120, heights around 64), 2-level pyramids (no level-2 window), gray
    frames, the first (no-motion) frame and both band sources."""
    for band_from_state in (1, 0):
        cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, lv)
        a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
        for p in (a, b):
            p.set_option("band_from_state", band_from_state)
            p.set_option("keep_float_output", 1)
        b.set_option("egress_strip", 0)
        for t in range(4):
            f = synth_frame(t, w, h, c)
            _, oa = a.process_image(f, cfg)
            _, ob = b.process_image(f, cfg)
            assert np.array_equal(oa, ob), (w, h, t, band_from_state, int(u8_diff(oa, ob).max()))
            assert np.array_equal(a.float_output(w, h, c), b.float_output(w, h, c)), (w, h, t)


@pytest.mark.parametrize("lanes,groups", [(8, 4), (5, 2), (3, 3), (16, 0), (2, 8)])
def test_lane_groups_equal_single_chain(lanes, groups):
    """Option lane_groups: the lanes of a handle run as several concurrent launch chains on their own CUDA streams (fork
    from / join into the handle's stream).  Every lane must come out bit-identical to the single-chain run — outputs,
    state planes, also after the group count changes mid-stream (state is kept) and through the pipelined host API."""
    w, h, lv = 200, 136, 4
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, lv)
    a, b = L.MagnificationProcessor(0, lanes=lanes), L.MagnificationProcessor(0, lanes=lanes)
    a.set_option("lane_groups", 1)
    b.set_option("lane_groups", groups)
    for t in range(6):
        f = np.stack([np.roll(synth_frame(t, w, h, 3), (3 * k, 7 * k), axis=(0, 1)) for k in range(lanes)])
        if t == 4:
            b.set_option("lane_groups", 2 if groups != 2 else 1)       # regroup mid-stream: temporal state must survive
        _, oa = a.process_image(f, cfg)
        _, ob = b.process_image(f, cfg)
        assert np.array_equal(oa, ob), (lanes, groups, t)
    for lvl in range(1, lv):
        for name in ("lowpassHi", "lowpassLo"):
            assert np.array_equal(a.get_state(name, lvl), b.get_state(name, lvl)), (lvl, name)


