"""mc_chain_geometry (no GPU): the geometry and *_is_input flags runChainOnce gives a frame, against the oracle's
run_chain_once with the magnifier off, over sizes, divisors (out-of-range ones clamp to 1..8), ROIs inside the frame, at
its edges and larger than it, gray on and off, and 1 and 3 channels."""
import itertools

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O

ROIS = [None, (0.2, 0.1, 0.5, 0.6), (0.999, 0.999, 0.5, 0.5), (0.0, 0.5, 1.0, 0.5), (0.6, 0.4, 1.7, 2.0), (-0.2, -0.1, 0.3, 0.3)]
SIZES = [(w, h) for w in range(1, 10) for h in range(1, 10)] + [(641, 479), (1921, 1079), (3839, 2161), (4095, 1), (1, 2159)]


def oracle_info(omag, w, h, c, down, roi, gray):
    ocfg = O.ProcessorConfig(grayscale=gray, preprocess=O.PreprocessParams(down, roi is not None, *(roi or (0.0, 0.0, 1.0, 1.0))),
                             magnification=O.MagnificationParams(mode=O.MODE_NONE))
    img = np.zeros((h, w) + ((3,) if c == 3 else ()), np.uint8)
    cur, orig, cur_same, orig_same = O.run_chain_once(omag, img, ocfg)
    g = lambda a: (0, 0, 0) if a is None else (a.shape[1], a.shape[0], 1 if a.ndim == 2 else a.shape[2])
    return (int(cur_same), *((0, 0, 0) if cur_same else g(cur)), int(orig_same), *((0, 0, 0) if orig_same else g(orig)), 0)


def geometry(w, h, c, down, roi, gray):
    cfg = L.ProcessorConfig(grayscale=gray, preprocess=L.PreprocessParams(down, roi is not None, *(roi or (0.0, 0.0, 1.0, 1.0))),
                            magnification=L.MagnificationParams(mode=L.MagnificationMode.NONE))
    i = L.ProcessingChainB200.geometry(cfg, w, h, c)
    return (i.cur_is_input, i.out_w, i.out_h, i.out_channels, i.orig_is_input, i.orig_w, i.orig_h, i.orig_channels, i.magnified)


@pytest.mark.parametrize("c,gray", [(3, False), (3, True), (1, False), (1, True)])
def test_geometry_matches_run_chain_once(built, c, gray):
    omag = O.MagnificationProcessor()
    for (w, h), down, roi in itertools.product(SIZES, range(0, 10), ROIS):
        assert geometry(w, h, c, down, roi, gray) == oracle_info(omag, w, h, c, down, roi, gray), (w, h, c, down, roi, gray)


def test_empty_frame_and_bad_arguments(built):
    import ctypes as C
    lib, p, info = capi.lib(), capi.McParams(), capi.McChainInfo()
    lib.mc_params_default(C.byref(p))
    p.pre_downscale = 2
    assert lib.mc_chain_geometry(C.byref(p), 0, 10, 3, 1, C.byref(info)) == capi.MC_OK
    assert (info.cur_is_input, info.orig_is_input, info.out_w, info.orig_w) == (1, 1, 0, 0)
    assert lib.mc_chain_geometry(C.byref(p), 10, 10, 2, 0, C.byref(info)) == capi.MC_ERR_INVALID
    assert lib.mc_chain_geometry(None, 10, 10, 3, 0, C.byref(info)) == capi.MC_ERR_INVALID
    assert lib.mc_chain_geometry(C.byref(p), 10, 10, 3, 0, None) == capi.MC_ERR_INVALID
