"""Pins the oracle (oracle/livim_oracle.py) against the reference's OWN hot-path code.

``oracle/_ref/_livim_ref`` is /root/reference/src/processing/** compiled unmodified (oracle/build_ref.py) against
the cvshim facade, whose pixel operations are the real OpenCV kernels in cv2.  Oracle and compiled reference are
fed the same frames and must agree BIT-EXACTLY: every u8 output, every passthrough decision, and the float
temporal state (EMA planes, rolling window, Riesz pyramids and IIR outputs).  CPU only.

Skipped only when the module is neither prebuilt nor buildable (no /root/reference and no oracle/_ref/*.so).
"""
import os

import numpy as np
import pytest

from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from oracle import livim_ref

R = livim_ref.load()
if R is None and os.environ.get("MC_REQUIRE_REF") == "1":
    raise RuntimeError("MC_REQUIRE_REF=1 but oracle/_ref/_livim_ref is missing")
pytestmark = pytest.mark.skipif(R is None, reason="oracle/_ref/_livim_ref is not built and /root/reference is absent")


def same(a, b):
    """bit-for-bit equality of two arrays (NaNs in the same places count as equal)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind == "f":
        return bool(np.array_equal(a, b, equal_nan=True))
    return bool(np.array_equal(a, b))


def cfg_pair(mode, amp, wl, lo, hi, chroma, levels, fps=30.0, **extra):
    """-> (reference ProcessorConfig built by the reference's own toParams, oracle ProcessorConfig)."""
    ui = R.MagUiValues()
    ui.mode = livim_ref.mode_enum(R, mode)
    ui.amplification, ui.wavelength, ui.low, ui.high, ui.chroma, ui.levels, ui.captureFps = amp, wl, lo, hi, chroma, levels, fps
    rc = R.ProcessorConfig()
    rc.magnification = R.toParams(ui)
    oc = O.ProcessorConfig(magnification=O.to_params(mode, amp, wl, lo, hi, chroma, levels, fps))
    for k in ("amplification", "coWavelength", "coLow", "coHigh", "chromAttenuation", "levels", "framerate"):
        assert getattr(rc.magnification, k) == getattr(oc.magnification, k), k   # toParams restated exactly
    for k, v in extra.items():
        if k == "grayscale":
            rc.grayscale = oc.grayscale = v
        else:
            pp = rc.preprocess
            setattr(pp, k, v)
            rc.preprocess = pp
            setattr(oc.preprocess, k, float(np.float32(v)) if isinstance(v, float) else v)
    return rc, oc


def run_pair(rc, oc, frames, rp=None, op=None):
    rp, op = rp or R.Processor(), op or O.MagnificationProcessor()
    for t, f in enumerate(frames):
        pr, ro = rp.process(f, rc)
        po, oo = op.process(f, oc)
        assert pr == po, f"frame {t}: produced {pr} (reference) vs {po} (oracle)"
        assert same(ro, oo if po else f), f"frame {t}: output differs"
    return rp, op


# --------------------------------------------------------------------------------------------------
# scalar / host functions
# --------------------------------------------------------------------------------------------------
def test_host_functions_are_bit_identical():
    for w in range(1, 70):
        for h in (1, 5, 6, 7, 11, 12, 13, 33, 64, 135, 1080):
            assert R.calculateMaxLevels(w, h) == O.calculate_max_levels(w, h)
    for sz in ((1920, 1080), (3840, 2160), (640, 480)):
        assert R.calculateMaxLevels(*sz) == O.calculate_max_levels(*sz)
    for fps in list(range(0, 130)) + [240, 1000]:
        assert R.getOptimalBufferSize(fps) == O.get_optimal_buffer_size(fps)
    for hz in (0.0, -1.0, 0.05, 0.4, 1.0, 3.0, 14.9, 15.0, 100.0):
        for fps in (30.0, 0.0, -5.0, 24.0, 59.94):
            assert R.motionHzToBlend(hz, fps) == O.motion_hz_to_blend(hz, fps)
    for wn in (0.4 / 15, 3.0 / 15, 0.8 / 15, 0.5, 0.9, 1e-3, 0.0):
        ra, rb = R.butterworth(2, wn)
        oa, ob = O.butterworth(2, wn)
        assert same(np.array(ra), np.array(oa)) and same(np.array(rb), np.array(ob)), wn


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_to_params_matches_reference(mode):
    for amp, wl, lo, hi, chroma, levels, fps in ((20, 50.0, 0.4, 3.0, 50, 6, 30.0), (100, 0.0, 0.8, 1.2, 0, 3, 24.0),
                                                 (7, 99.5, 0.0, 14.0, 100, 1, 60.0)):
        cfg_pair(mode, amp, wl, lo, hi, chroma, levels, fps)


# --------------------------------------------------------------------------------------------------
# Motion (Laplace)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,c,levels,chroma", [(96, 64, 3, 4, 50), (97, 67, 3, 3, 0), (131, 75, 1, 4, 0), (64, 48, 3, 9, 100)])
def test_laplace_outputs_and_state_bit_exact(w, h, c, levels, chroma):
    rc, oc = cfg_pair(0, 20, 50.0, 0.4, 3.0, chroma, levels)
    core, st = R.Core(), O.MotionState()
    lv = min(max(levels, 1), O.calculate_max_levels(w, h))
    for t in range(7):
        f = synth_frame(t, w, h, c)
        pr, ro = core.run(0, f, rc.magnification, lv)
        po, oo = O.magnify_motion(f, oc.magnification, lv, c, st)
        assert pr and po and same(ro, oo), t
        hi, lo = core.motion_state()
        assert len(hi) == len(st.lowpassHi) == lv + 1
        for l in range(lv + 1):
            assert same(hi[l], st.lowpassHi[l]) and same(lo[l], st.lowpassLo[l]), (t, l)
    # the same through MagnificationProcessor (levels clamp + tracker)
    run_pair(rc, oc, [synth_frame(t, w, h, c) for t in range(5)])


def test_laplace_live_parameter_changes_resets_and_passthrough():
    w, h = 80, 60
    frames = [synth_frame(t, w, h, 3) for t in range(12)]
    rc, oc = cfg_pair(0, 20, 50.0, 0.4, 3.0, 30, 3)
    rp, op = run_pair(rc, oc, frames[:4])
    rc2, oc2 = cfg_pair(0, 45, 20.0, 0.0, 5.0, 80, 3)          # non-structural: alpha, wavelength, cutoffs (coLow = 0), chroma
    run_pair(rc2, oc2, frames[4:7], rp, op)
    rc3, oc3 = cfg_pair(0, 45, 20.0, 0.0, 5.0, 80, 2)          # structural: levels -> state reset
    run_pair(rc3, oc3, frames[7:9], rp, op)
    run_pair(rc3, oc3, [synth_frame(t, 70, 50, 3) for t in range(3)], rp, op)   # structural: size
    run_pair(rc3, oc3, [synth_frame(t, 70, 50, 1) for t in range(3)], rp, op)   # structural: channels
    rcn, ocn = cfg_pair(3, 45, 20.0, 0.0, 5.0, 80, 2)          # mode None: identity, frees state
    run_pair(rcn, ocn, frames[9:10], rp, op)
    run_pair(rc3, oc3, frames[10:12], rp, op)
    rp.reset(); op.reset()
    run_pair(rc3, oc3, frames[:2], rp, op)
    run_pair(rc, oc, [synth_frame(0, 5, 40, 3), synth_frame(1, 40, 5, 3), synth_frame(2, 6, 6, 3)], rp, op)   # <= 5 px: identity


def test_laplace_1080p_config2_first_frames():
    """BASELINE.json configs[1] (1920x1080x3, 6 levels) — the bench workload — two frames, bit-exact."""
    rc, oc = cfg_pair(0, 20, 50.0, 0.4, 3.0, 0, 6)
    run_pair(rc, oc, [synth_frame(t, 1920, 1080, 3) for t in range(2)])


# --------------------------------------------------------------------------------------------------
# Color (Gaussian + ideal FFT)
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,c,levels,fps", [(96, 64, 3, 3, 8.0), (90, 70, 1, 2, 8.0), (64, 48, 3, 2, 12.0)])
def test_color_warmup_wraparound_and_window_bit_exact(w, h, c, levels, fps):
    rc, oc = cfg_pair(2, 100, 0.0, 0.8, 1.2, 0, levels, fps)
    core, st = R.Core(), O.ColorState()
    n = O.get_optimal_buffer_size(int(fps)) + 5      # every DFT length 2..cap (odd ones included), then the shift
    for t in range(n):
        f = synth_frame(t, w, h, c, fps=fps)
        pr, ro = core.run(2, f, rc.magnification, levels)
        po, oo = O.magnify_color(f, oc.magnification, levels, c, st)
        assert pr == po == (t >= 1), t
        if pr:
            assert same(ro, oo), t
        win = core.color_window()
        ow = st.window if c > 1 else st.window[:, :, 0]
        assert same(win, ow), t


def test_color_framerate_change_and_zero_low_cutoff():
    w, h = 72, 56
    rc, oc = cfg_pair(2, 60, 0.0, 0.0, 1.5, 0, 2, 12.0)        # coLow == 0 -> 0.01 Hz
    rp, op = run_pair(rc, oc, [synth_frame(t, w, h, 3) for t in range(20)])
    rc2, oc2 = cfg_pair(2, 60, 0.0, 0.0, 1.5, 0, 2, 8.0)       # smaller cap mid-stream (window shrinks by one per frame)
    run_pair(rc2, oc2, [synth_frame(20 + t, w, h, 3) for t in range(12)], rp, op)


# --------------------------------------------------------------------------------------------------
# Phase (Riesz)
# --------------------------------------------------------------------------------------------------
RIESZ_PLANES = (("lowpass", lambda l: l.lowpass), ("rx", lambda l: l.rx), ("ry", lambda l: l.ry),
                ("amplitude", lambda l: l.amplitude), ("amplitude_blurred", lambda l: l.amplitude_blurred),
                ("phase_diff_cos", lambda l: l.phase_diff[0]), ("phase_diff_sin", lambda l: l.phase_diff[1]))
RIESZ_IIR = (("lowpass_iir_cos", lambda l: l.lowpass_iir[0]), ("lowpass_iir_sin", lambda l: l.lowpass_iir[1]),
             ("highpass_iir_cos", lambda l: l.highpass_iir[0]), ("highpass_iir_sin", lambda l: l.highpass_iir[1]))


@pytest.mark.parametrize("w,h,levels", [(96, 64, 3), (101, 77, 4)])
def test_riesz_outputs_and_every_state_plane_bit_exact(w, h, levels):
    rc, oc = cfg_pair(1, 50, 50.0, 0.4, 3.0, 0, levels)
    core, st = R.Core(), O.RieszState()
    for t in range(6):
        f = synth_frame(t, w, h, 3)
        pr, ro = core.run(1, f, rc.magnification, levels)
        po, oo = O.magnify_riesz(f, oc.magnification, levels, 3, st)
        assert pr == po == (t >= 1), t
        if not pr:
            continue
        assert same(ro, oo), t
        for which, opyr in ((True, st.old), (False, st.cur)):
            for l, (rl, ol) in enumerate(zip(core.riesz_levels(which), opyr.levels)):
                for name, get in RIESZ_PLANES + (() if which else RIESZ_IIR):
                    ov = get(ol)
                    assert (rl[name] is None) == (ov is None) or ov is None or rl[name] is None, (t, which, l, name)
                    if rl[name] is not None and ov is not None:
                        assert same(rl[name], ov), (t, "old" if which else "cur", l, name)
    ra = core.riesz_coefficients()
    assert ra[0] == st.lo.A and ra[1] == st.lo.B and ra[2] == st.hi.A and ra[3] == st.hi.B


def test_riesz_cutoff_change_gray_passthrough_and_processor():
    w, h = 88, 66
    frames = [synth_frame(t, w, h, 3) for t in range(10)]
    rc, oc = cfg_pair(1, 50, 50.0, 0.4, 3.0, 0, 3)
    rp, op = run_pair(rc, oc, frames[:4])
    rc2, oc2 = cfg_pair(1, 35, 70.0, 0.8, 3.0, 0, 3)           # low cutoff changes: redesign + register reset + old rebuilt
    run_pair(rc2, oc2, frames[4:6], rp, op)
    rc3, oc3 = cfg_pair(1, 35, 70.0, 0.8, 2.0, 0, 3)           # high cutoff changes
    run_pair(rc3, oc3, frames[6:8], rp, op)
    rc4, oc4 = cfg_pair(1, 35, 70.0, 0.8, 2.0, 0, 3, 25.0)     # framerate alone: coefficients are NOT recomputed
    run_pair(rc4, oc4, frames[8:10], rp, op)
    run_pair(rc, oc, [synth_frame(t, w, h, 1) for t in range(3)])   # gray input: silent passthrough


# --------------------------------------------------------------------------------------------------
# Front of the chain (SURVEY 8f-1): PreprocessProcessor -> GrayscaleProcessor -> MagnificationProcessor
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [
    dict(downscale=2), dict(downscale=4, grayscale=True), dict(downscale=8),
    dict(roiEnabled=True, roiX=0.1, roiY=0.2, roiW=0.55, roiH=0.6),
    dict(roiEnabled=True, roiX=0.13, roiY=0.07, roiW=0.61, roiH=0.77, downscale=2, grayscale=True),
    dict(roiEnabled=True, roiX=0.9, roiY=0.9, roiW=0.5, roiH=0.5, downscale=4),    # clamped to the frame
    dict(grayscale=True), dict(),
])
def test_chain_bit_exact(extra):
    w, h = 203, 151
    rc, oc = cfg_pair(0, 20, 50.0, 0.4, 3.0, 40, 3, **extra)
    chain, omag = R.Chain(), O.MagnificationProcessor()
    for t in range(4):
        f = synth_frame(t, w, h, 3)
        rcur, rorig, r_cur_is_in, r_orig_is_in, _gray = chain.process(f, rc)
        ocur, oorig, o_cur_is_in, o_orig_is_in = O.run_chain_once(omag, f, oc)
        assert r_cur_is_in == o_cur_is_in and r_orig_is_in == o_orig_is_in, t
        assert same(rorig, oorig) and same(rcur, ocur), t


# --------------------------------------------------------------------------------------------------
# The drop-in: reference chain + reference headers + the product's adapter (needs an H100 to run)
# --------------------------------------------------------------------------------------------------
def test_dropin_chain_builds_against_real_reference_headers_and_has_no_cpu_fallback(built):
    """oracle/_ref/_livim_ref also holds the reference's chain with the ONE substitution of INTEGRATION.md
    (MagnificationProcessorB200 at ChainBuilder.cpp:15), compiled against the reference's real IProcessor.hpp /
    Frame.hpp.  Without a GPU constructing it must fail loudly: mc_create reports no device, the adapter throws."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by tests/test_gpu_vs_reference.py::test_dropin_chain_on_gpu")
    R.set_magcore_library(built[0])
    with pytest.raises(RuntimeError, match="magcore_b200"):
        R.DropInChain(0)
