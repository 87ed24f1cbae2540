"""Kernel-LOGIC regression on the CUDA-on-CPU emulation (tests/cuda_emu) — no GPU, no product library compute.

The product's own kernel sources are compiled with g++ against an emulated CUDA runtime (CTA threads as cooperative
fibers, emulated TMA / mbarrier / shuffles / cuFFT) into tests/cuda_emu/libmagcore_emu.so, and tiny clips of all
three modes plus the fused front of the chain are checked against the oracle with the same tolerances as the
`-m gpu` parity tests.  This catches indexing / border / staging / state-handling regressions in the kernels on
a machine without a GPU; it says nothing about performance or hardware behaviour — the `-m gpu` tests on an H100
remain the parity gate.  The whole `-m gpu` suite can be pointed at the emulation with `MC_EMU=1` (tests/conftest.py).
"""
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs, u8_diff

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def run_mode(mode, ui, w, h, c, n, fps=30.0, options=()):
    cfg, ocfg = make_cfgs(mode, *ui, fps)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    for k, v in options:
        proc.set_option(k, v)
    worst, same = 0, []
    for t in range(n):
        f = synth_frame(t, w, h, c, fps=fps)
        produced, out = proc.process_image(f, cfg)
        oprod, oout = oproc.process(f, ocfg)
        assert produced == oprod, t
        if produced:
            d = u8_diff(out, oout)
            worst = max(worst, int(d.max()))
            same.append(float((d == 0).mean()))
    proc.close()
    return worst, min(same)


@pytest.mark.parametrize("w,h,c,levels,tma", [(131, 75, 3, 4, 1), (131, 75, 3, 4, 0), (96, 67, 1, 3, 1)])
def test_laplace_kernels_on_emulation(emu, w, h, c, levels, tma):
    worst, _ = run_mode(O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 40, levels), w, h, c, 5, options=(("use_tma", tma),))
    assert worst <= 1


def test_color_kernels_on_emulation(emu):
    worst, _ = run_mode(O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 2), 90, 66, 3, 19, fps=8.0)   # all DFT lengths 2..16 + wrap
    assert worst <= 1


def test_riesz_kernels_on_emulation(emu):
    worst, same = run_mode(O.MODE_PHASE, (50, 50.0, 0.4, 3.0, 0, 3), 120, 90, 3, 5)
    assert worst <= 3 and same >= 0.995


def test_chain_front_stages_on_emulation(emu):
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 20, 3)
    cfg.grayscale = ocfg.grayscale = True
    cfg.preprocess = L.PreprocessParams(3, True, 0.1, 0.2, 0.77, 0.61)      # fractional INTER_AREA scale + ROI + gray
    ocfg.preprocess = O.PreprocessParams(3, True, 0.1, 0.2, 0.77, 0.61)
    chain, omag = L.ProcessingChainB200(0), O.MagnificationProcessor()
    for t in range(3):
        f = synth_frame(t, 203, 151, 3)
        cur, orig = chain.run_chain_once(L.Frame(image=f, seq=t), cfg)
        ocur, oorig, _, _ = O.run_chain_once(omag, f, ocfg)
        assert np.array_equal(orig.image, oorig), t
        assert int(u8_diff(cur.image, ocur).max()) <= 1, t


@pytest.mark.parametrize("env", [{}, {"CUDA_EMU_ORDER": "reverse"}, {"CUDA_EMU_ORDER": "random"}, {"CUDA_EMU_ASYNC": "1"},
                                 {"CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "5"}],
                         ids=["default", "reverse", "random", "async", "async+random"])
def test_emulation_selftest(env):
    """The emulation itself against closed forms (tests/cuda_emu/selftest): warp shuffles with lanes that exit after
    taking part, barriers with exited threads, two TMA loads (one partly out of bounds) on one mbarrier with transaction
    counting, the tensor-map encoder's alignment rules, atomics, and a producer/consumer pair on two streams — which must
    be right with its event wait in every mode and observably wrong without it when streams run asynchronously."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    d = os.path.join(root, "tests", "cuda_emu", "selftest")
    exe = os.path.join(d, "selftest")
    srcs = [os.path.join(d, "selftest.cpp"), os.path.join(root, "tests", "cuda_emu", "emu_runtime.cpp")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-I", os.path.join(root, "tests", "cuda_emu", "include"), *srcs, "-o", exe],
                       check=True)
    r = subprocess.run([exe], env={**os.environ, **env}, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "selftest: ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_exception_inside_a_frame_is_contained_and_resets_state(emu):
    """A C++ exception thrown while a frame is being processed (std::bad_alloc injected at the top of the device-side
    body) comes back as MC_ERR_INTERNAL, drops the temporal state (the recovery contract of
    ProcessingChain.cpp:50-62) and leaves the handle usable: the next frames equal a fresh stream's."""
    import ctypes as C
    lib = capi.lib()
    lib.mc_debug_inject_exception.argtypes = [C.c_int]
    lib.mc_debug_inject_exception.restype = None
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 3)
    proc = L.MagnificationProcessor(0)
    for t in range(3):
        proc.process_image(synth_frame(t, 80, 60, 3), cfg)
    lib.mc_debug_inject_exception(1)
    with pytest.raises(L.MagcoreError) as e:
        proc.process_image(synth_frame(3, 80, 60, 3), cfg)
    assert e.value.status == capi.MC_ERR_INTERNAL and "bad_alloc" in str(e.value)
    oproc = O.MagnificationProcessor()                       # the stream restarts from scratch after the failure
    for t in range(4, 7):
        f = synth_frame(t, 80, 60, 3)
        produced, out = proc.process_image(f, cfg)
        oprod, oout = oproc.process(f, ocfg)
        assert produced == oprod and int(u8_diff(out, oout).max()) <= 1
    proc.close()


def test_color_many_lanes_and_frame_rate_sweep(emu):
    """ADVICE r1: (1) the per-lane min/max scratch must be initialised for EVERY lane (lanes > 64 used to read
    uninitialised slots); (2) sweeping the frame rate up and down re-lays the ring out once per change (no per-frame
    compaction, no leaked buffers) and still matches the reference's window semantics."""
    lanes, w, h = 70, 24, 20
    cfg, ocfg = make_cfgs(O.MODE_COLOR, 60, 0.0, 0.8, 1.2, 0, 1, 8.0)
    proc = L.MagnificationProcessor(0, lanes=lanes)
    oprocs = {k: O.MagnificationProcessor() for k in (0, 63, 64, 69)}
    for t in range(6):
        clip = np.stack([np.roll(synth_frame(t, w, h, 3, fps=8.0), (k, 2 * k), axis=(0, 1)) for k in range(lanes)])
        produced, out = proc.process_image(clip, cfg)
        for k, op in oprocs.items():
            oprod, oout = op.process(clip[k], ocfg)
            assert produced == oprod
            if produced:
                assert int(u8_diff(out[k], oout).max()) <= 1, (t, k)
    proc.close()
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    t = 0
    for fps in (8.0, 30.0, 8.0, 4.0, 16.0):          # caps 16 -> 64 -> 16 -> 8 -> 32, partly and fully filled windows
        cfg, ocfg = make_cfgs(O.MODE_COLOR, 60, 0.0, 0.8, 1.2, 0, 1, fps)
        for _ in range(11):
            f = synth_frame(t, 40, 30, 3, fps=8.0)
            produced, out = proc.process_image(f, cfg)
            oprod, oout = oproc.process(f, ocfg)
            assert produced == oprod, (fps, t)
            if produced:
                assert int(u8_diff(out, oout).max()) <= 1, (fps, t)
            t += 1
    proc.close()


def test_round2_kernel_forms_agree_on_emulation(emu):
    """Round-2 kernel forms, logic only (the H100 runs the same checks in test_gpu_laplace.py / test_gpu_riesz.py):
    (1) the shuffle-strip egress equals the shared-memory tile egress bit for bit over several strips and chunks, both band
    sources, float taps included; (2) lanes run as two launch chains (option lane_groups) equal one chain; (3) the 9x9 Riesz
    kernels give the same bits with TMA-staged and with LDG-staged tiles."""
    w, h, lv = 250, 131, 3
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, lv)
    for bfs in (1, 0):
        a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
        for p in (a, b):
            p.set_option("band_from_state", bfs)
            p.set_option("keep_float_output", 1)
        b.set_option("egress_strip", 0)
        for t in range(3):
            f = synth_frame(t, w, h, 3)
            _, oa = a.process_image(f, cfg)
            _, ob = b.process_image(f, cfg)
            assert np.array_equal(oa, ob), (bfs, t)
            assert np.array_equal(a.float_output(w, h, 3), b.float_output(w, h, 3)), (bfs, t)
        a.close(); b.close()
    lanes = 5
    a, b = L.MagnificationProcessor(0, lanes=lanes), L.MagnificationProcessor(0, lanes=lanes)
    a.set_option("lane_groups", 1)
    b.set_option("lane_groups", 2)
    for t in range(3):
        f = np.stack([np.roll(synth_frame(t, 130, 70, 3), (3 * k, 7 * k), axis=(0, 1)) for k in range(lanes)])
        _, oa = a.process_image(f, cfg)
        _, ob = b.process_image(f, cfg)
        assert np.array_equal(oa, ob), t
    a.close(); b.close()
    cfgp, _ = make_cfgs(O.MODE_PHASE, 40, 50.0, 0.4, 3.0, 0, 3, 30.0)
    a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
    b.set_option("use_tma", 0)
    for t in range(3):
        f = synth_frame(t, 230, 120, 3)
        pa, oa = a.process_image(f, cfgp)
        pb, ob = b.process_image(f, cfgp)
        assert pa == pb and (not pa or np.array_equal(oa, ob)), t
    a.close(); b.close()


def test_riesz_band_planes_bit_identical_on_odd_widths_on_emulation(emu):
    """mc_riesz.cu::f2d — cv::filter2D's FMA / multiply-then-add column rule: band planes and Riesz pair equal the
    oracle's bit for bit on a width that is not a multiple of 8 (the H100 runs the same check in test_gpu_riesz.py)."""
    w, h, levels = 71, 76, 4
    cfg, ocfg = make_cfgs(O.MODE_PHASE, 50, 50.0, 0.4, 3.0, 0, levels, 30.0)
    proc, op = L.MagnificationProcessor(0), O.MagnificationProcessor()
    for t in range(3):
        f = synth_frame(t, w, h, 3)
        _, out = proc.process_image(f, cfg)
        _, oout = op.process(f, ocfg)
    assert np.array_equal(out, oout)                       # libm on both sides: the whole frame is identical here
    for lvl in range(levels - 1):
        ref = op.riesz.old.levels[lvl]
        for name, plane in (("old.lowpass", ref.lowpass), ("old.rx", ref.rx), ("old.ry", ref.ry)):
            assert np.array_equal(proc.get_state(name, lvl)[0, 0], np.asarray(plane)), (name, lvl)
    proc.close()
