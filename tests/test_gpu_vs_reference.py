"""CUDA path (through the C ABI) checked DIRECTLY against the reference's own code on the GPU.

The checker here is not the oracle restatement but oracle/_ref/_livim_ref: /root/reference/src/processing/**
compiled unmodified (oracle/build_ref.py, prebuilt under oracle/_ref/ where the reference sources are present) with OpenCV's
kernels underneath.  Same tolerances as the oracle-based tests: Laplace / Color <= 1 LSB free-running,
Phase <= 3 LSB and >= 99.5 % identical free-running; passthrough decisions identical."""
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from oracle import livim_ref
from common import make_cfgs, u8_diff

import os

R = livim_ref.load()
if R is None and os.environ.get("MC_REQUIRE_REF") == "1":
    # a GPU run must not silently lose its reference-pinned tests
    raise RuntimeError("MC_REQUIRE_REF=1 but oracle/_ref/_livim_ref is missing: run __graft_entry__.build() where "
                       "the reference sources are present, and keep oracle/_ref/ with the tree")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(R is None, reason="oracle/_ref/_livim_ref not present")]


def pair(mode, amp, wl, lo, hi, chroma, levels, fps=30.0):
    cfg, ocfg = make_cfgs(mode, amp, wl, lo, hi, chroma, levels, fps)
    return cfg, livim_ref.to_ref_config(R, ocfg)


@pytest.mark.parametrize("w,h,c,levels,chroma", [(320, 240, 3, 4, 50), (640, 480, 3, 4, 0), (241, 135, 1, 5, 0), (1920, 1080, 3, 6, 0)])
def test_laplace_vs_compiled_reference(w, h, c, levels, chroma):
    cfg, rcfg = pair(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, chroma, levels)
    proc, ref = L.MagnificationProcessor(0), R.Processor()
    for t in range(6 if w > 1000 else 16):
        f = synth_frame(t, w, h, c)
        produced, out = proc.process_image(f, cfg)
        rprod, rout = ref.process(f, rcfg)
        assert produced == rprod, t
        assert int(u8_diff(out, rout).max()) <= 1, t


def test_color_vs_compiled_reference():
    cfg, rcfg = pair(O.MODE_COLOR, 100, 0.0, 0.8, 1.2, 0, 3, 8.0)
    proc, ref = L.MagnificationProcessor(0), R.Processor()
    for t in range(24):   # every warm-up DFT length up to the 16-column cap, then the rolling window
        f = synth_frame(t, 320, 240, 3, fps=8.0)
        produced, out = proc.process_image(f, cfg)
        rprod, rout = ref.process(f, rcfg)
        assert produced == rprod, t
        if produced:
            assert int(u8_diff(out, rout).max()) <= 1, t


def test_phase_vs_compiled_reference():
    cfg, rcfg = pair(O.MODE_PHASE, 50, 50.0, 0.4, 3.0, 0, 4)
    proc, ref = L.MagnificationProcessor(0), R.Processor()
    for t in range(12):
        f = synth_frame(t, 480, 270, 3)
        produced, out = proc.process_image(f, cfg)
        rprod, rout = ref.process(f, rcfg)
        assert produced == rprod, t
        if produced:
            d = u8_diff(out, rout)
            assert int(d.max()) <= 3 and float((d == 0).mean()) >= 0.995, (t, int(d.max()), float((d == 0).mean()))


def test_chain_vs_compiled_reference():
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 20, 4)
    cfg.grayscale = ocfg.grayscale = True
    cfg.preprocess = L.PreprocessParams(2, True, 0.1, 0.2, 0.77, 0.61)
    ocfg.preprocess = O.PreprocessParams(2, True, 0.1, 0.2, 0.77, 0.61)
    rcfg = livim_ref.to_ref_config(R, ocfg)
    chain, rchain = L.ProcessingChainB200(0), R.Chain()
    for t in range(5):
        f = synth_frame(t, 641, 479, 3)
        cur, orig = chain.run_chain_once(L.Frame(image=f, seq=t), cfg)
        rcur, rorig, _cur_same, _orig_same, _gray = rchain.process(f, rcfg)
        assert np.array_equal(orig.image, rorig), t                 # integer front stages: bit-exact
        assert cur.image.shape == rcur.shape and int(u8_diff(cur.image, rcur).max()) <= 1, t


def test_dropin_chain_on_gpu():
    """The drop-in as a maintainer would build it: the reference's PreprocessProcessor and GrayscaleProcessor
    (compiled reference code), MagnificationProcessorB200 (the product's adapter, compiled against the real
    reference headers) as the third stage, driven by the reference's runChainOnce — against the all-reference chain."""
    from lvm_b200 import capi
    R.set_magcore_library(capi.LIB_PATH)   # libmagcore_b200.so (tests/cuda_emu's build when MC_EMU=1)
    for mode, ui, gray, pre in ((O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 30, 4), False, (2, True, 0.1, 0.1, 0.8, 0.8)),
                                (O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 3), True, (1, False, 0.0, 0.0, 1.0, 1.0)),
                                (O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 2), False, (4, False, 0.0, 0.0, 1.0, 1.0)),
                                (O.MODE_PHASE, (50, 50.0, 0.4, 3.0, 0, 3), False, (2, False, 0.0, 0.0, 1.0, 1.0))):
        _, ocfg = make_cfgs(mode, *ui)
        ocfg.grayscale = gray
        ocfg.preprocess = O.PreprocessParams(*pre)
        rcfg = livim_ref.to_ref_config(R, ocfg)
        dropin, ref = R.DropInChain(0), R.Chain()
        for t in range(8):
            f = synth_frame(t, 640, 480, 3)
            cur, orig, cur_is_in, orig_is_in, is_gray = dropin.process(f, rcfg)
            rcur, rorig, rcur_is_in, rorig_is_in, ris_gray = ref.process(f, rcfg)
            assert (cur_is_in, orig_is_in, is_gray) == (rcur_is_in, rorig_is_in, ris_gray), (mode, t)
            assert np.array_equal(orig, rorig), (mode, t)
            d = u8_diff(cur, rcur)
            if mode == O.MODE_PHASE:
                assert int(d.max()) <= 3 and float((d == 0).mean()) >= 0.995, (t, int(d.max()))
            else:
                assert int(d.max()) <= 1, (mode, t, int(d.max()))
        dropin.reset()
