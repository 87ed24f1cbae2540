"""CPU tests of the host side: C-ABI exports, parameter mapping, scalar design code, and the product's
per-pixel __host__ __device__ functions compiled for the CPU (tests/hostcheck) against cv2."""
import ctypes as C
import os
import re

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hc(built):
    lib = C.CDLL(built[1])
    return lib


def test_library_exports_every_declared_symbol(built):
    hdr = open(os.path.join(ROOT, "include", "magcore_b200.h")).read()
    declared = set(re.findall(r"\b(mc_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"mc_status", "mc_mode", "mc_params", "mc_handle", "mc_chain_info"}
    lib = C.CDLL(built[0])
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert declared == set(capi.SIGNATURES), declared ^ set(capi.SIGNATURES)
    assert lib.mc_abi_version() == 2
    assert hasattr(lib, "mc_debug_inject_exception")   # test hook, deliberately not in the public header


def test_no_cpu_fallback_without_gpu(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(L.MagcoreError) as e:
        L.MagnificationProcessor(0)
    assert e.value.status == capi.MC_ERR_NO_DEVICE


def test_params_mapping_matches_reference_formulas(built):
    for mode in (0, 1, 2):
        for amp, wl, lo, hi, chroma, lv, fps in [(20, 50.0, 0.4, 3.0, 0, 6, 30.0), (50, 30.0, 1.0, 5.0, 25, 4, 25.0),
                                                  (100, 80.0, 0.0, 1.2, 100, 3, 0.0), (10, 10.0, 14.9, 15.0, 7, 2, 30.0)]:
            a = L.toParams(L.MagUiValues(L.MagnificationMode(mode), amp, wl, lo, hi, chroma, lv, fps))
            b = O.to_params(mode, amp, wl, lo, hi, chroma, lv, fps)
            for k in ("amplification", "coWavelength", "coLow", "coHigh", "chromAttenuation", "levels", "framerate"):
                assert getattr(a, k) == getattr(b, k), (mode, k)


def test_max_levels_and_buffer_size(built):
    for w, h in [(1920, 1080), (640, 480), (3840, 2160), (6, 6), (5, 100), (7, 9), (130, 66), (1, 1), (4096, 6)]:
        assert L.calculateMaxLevels(w, h) == O.calculate_max_levels(w, h)
    assert (L.calculateMaxLevels(640, 480), L.calculateMaxLevels(1920, 1080), L.calculateMaxLevels(3840, 2160)) == (7, 8, 9)
    for fps in (0, 1, 7, 8, 9, 24, 25, 30, 32, 33, 60, 120, 240):
        assert L.getOptimalBufferSize(fps) == O.get_optimal_buffer_size(fps)


def test_butterworth_matches_oracle_and_scipy(built):
    from scipy.signal import butter
    for wn in (0.4 / 15, 3.0 / 15, 0.8 / 15, 0.01, 0.5, 0.9):
        a, b = L.butterworth(2, wn)
        oa, ob = O.butterworth(2, wn)
        sb, sa = butter(2, wn)
        assert np.allclose(a, oa, rtol=0, atol=1e-13) and np.allclose(b, ob, rtol=0, atol=1e-13)
        assert np.allclose(a, sa, rtol=0, atol=1e-13) and np.allclose(b, sb, rtol=0, atol=1e-13)
    a, b = L.butterworth(4, 0.3)
    sb, sa = butter(4, 0.3)
    assert np.allclose(a, sa, atol=1e-12) and np.allclose(b, sb, atol=1e-12)


def test_motion_gains_bit_identical(built):
    lib = capi.lib()
    for (w, h, lv, amp, wl) in [(1920, 1080, 6, 20, 50.0), (640, 480, 4, 20, 50.0), (3840, 2160, 8, 20, 50.0),
                                (320, 240, 4, 35, 20.0), (100, 100, 3, 0, 0.0), (200, 100, 5, 150, 100.0)]:
        p = capi.McParams()
        lib.mc_params_from_ui(C.byref(p), 0, amp, wl, 0.4, 3.0, 0, lv, 30.0)
        g = (C.c_float * (lv + 1))()
        assert lib.mc_motion_gains(C.byref(p), lv, w, h, g) == 0
        ref = O.motion_gains(O.to_params(0, amp, wl, 0.4, 3.0, 0, lv, 30.0), lv, w, h)
        assert [np.float32(x) for x in g] == [np.float32(x) for x in ref]
    # SURVEY §8d config 2 gains
    ref = O.motion_gains(O.to_params(0, 20, 50.0, 0.4, 3.0, 0, 6, 30.0), 6, 1920, 1080)
    assert np.allclose(ref, [0, -0.0725, 1.855, 5.710, 13.420, 20, 0], atol=2e-3)


def all_colours():
    """Every 24-bit colour once, as (b, g, r) = (i >> 16, (i >> 8) & 255, i & 255)."""
    i = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8)


def test_bgr2lab_device_function_is_bit_exact_with_cv2(hc):
    """Every colour: this pins the whole LUT, including the clamped neighbours at the top of the lattice."""
    assert hc.hc_lut_entries() == 34 * 33 * 33   # LabLutCell table: one padded b slab
    edge = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 255, 0], [0, 0, 255], [8, 8, 8], [7, 9, 247]], np.uint8)
    px = np.concatenate([all_colours(), edge])
    got = np.empty((len(px), 3), np.float32)
    hc.hc_bgr_to_lab(px.ctypes.data_as(C.c_void_p), len(px), got.ctypes.data_as(C.c_void_p))
    ref = cv2.cvtColor((px.astype(np.float32) * np.float32(1 / 255.0))[None], cv2.COLOR_BGR2Lab)[0]
    assert np.array_equal(got, ref)


def test_lab2bgr_device_function_matches_cv2(hc):
    rng = np.random.default_rng(1)
    px = all_colours()
    lab = cv2.cvtColor((px.astype(np.float32) * np.float32(1 / 255.0))[None], cv2.COLOR_BGR2Lab)[0]
    lab = np.concatenate([lab, lab[rng.integers(0, len(lab), 40000)] + rng.normal(0, 4, (40000, 3)).astype(np.float32),
                          np.stack([rng.uniform(-10, 110, 5000), rng.uniform(-150, 150, 5000), rng.uniform(-150, 150, 5000)], -1).astype(np.float32)])
    lab = np.ascontiguousarray(lab, np.float32)
    got = np.empty_like(lab)
    hc.hc_lab_to_bgr(lab.ctypes.data_as(C.c_void_p), len(lab), got.ctypes.data_as(C.c_void_p))
    ref = cv2.cvtColor(lab[None], cv2.COLOR_Lab2BGR)[0]
    assert float(np.abs(got - ref).max()) < 2e-5
    # non-finite L (Phase mode: 0/0 in flat regions, SURVEY A.6-9): OpenCV's clip max(min(v,1),0) turns NaN into 1.0
    odd = np.array([[np.nan, 0, 0], [np.nan, 40, -30], [np.inf, 0, 0], [-np.inf, 5, 5], [1e30, 0, 0], [-1e30, 0, 0]], np.float32)
    odd = np.ascontiguousarray(np.tile(odd, (3, 1)))
    got = np.empty_like(odd)
    hc.hc_lab_to_bgr(odd.ctypes.data_as(C.c_void_p), len(odd), got.ctypes.data_as(C.c_void_p))
    assert np.array_equal(got, cv2.cvtColor(odd[None], cv2.COLOR_Lab2BGR)[0])


def test_u8_quantiser_and_ema_match_oracle_helpers(hc):
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.uniform(-0.2, 1.2, 100000), np.arange(0, 256) / 255.0, (np.arange(0, 256) + 0.5) / 255.0,
                        [np.nan, np.inf, -np.inf]]).astype(np.float32)
    got = np.empty(len(x), np.uint8)
    hc.hc_unit_to_u8(x.ctypes.data_as(C.c_void_p), len(x), got.ctypes.data_as(C.c_void_p))
    with np.errstate(all="ignore"):
        ref = O._f32_to_u8(x, 255.0, 1.0 / 255.0)
    assert np.array_equal(got, ref)          # non-finite and huge inputs included (NaN, +-inf -> 0: cvtps2dq semantics)
    huge = np.array([1e7, 8.0e6, 3e9, -3e9, 2147483648.0 / 255.0 + 1.0], np.float32)
    got_h = np.empty(len(huge), np.uint8)
    hc.hc_unit_to_u8(huge.ctypes.data_as(C.c_void_p), len(huge), got_h.ctypes.data_as(C.c_void_p))
    assert np.array_equal(got_h, O._f32_to_u8(huge, 255.0, 1.0 / 255.0)) and got_h.tolist() == [0, 255, 0, 0, 0]
    s = rng.normal(0, 30, 100000).astype(np.float32)
    v = rng.normal(0, 30, 100000).astype(np.float32)
    out = np.empty_like(s)
    hc.hc_ema.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    c = 0.4665119089088967
    hc.hc_ema(s.ctypes.data, v.ctypes.data, len(s), c, out.ctypes.data)
    ref = cv2.addWeighted(s, 1 - c, v, c, 0).ravel()
    assert np.mean(out == ref) > 0.9999 and np.abs(out - ref).max() < 1e-5


def test_gaussian_taps(hc):
    t = np.empty(13, np.float32)
    hc.hc_gauss13(t.ctypes.data_as(C.c_void_p))
    assert np.array_equal(t, cv2.getGaussianKernel(13, 3.0, cv2.CV_32F).ravel())


def test_cpp_adapter_compiles_and_refuses_without_gpu(built):
    """adapter/MagnificationProcessorB200.hpp (the reference-side IProcessor) builds against stub reference
    headers; with no GPU its constructor must throw (rc 3) — there is no CPU fallback."""
    import subprocess
    import torch
    exe = os.path.join(ROOT, "tests", "adapter_stub", "adapter_check")
    if not os.path.exists(exe):
        import __graft_entry__ as g
        g.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    if torch.cuda.is_available():
        assert r.returncode == 0 and "OK gpu" in r.stdout, r.stdout
    else:
        assert r.returncode == 3 and "no usable CUDA device" in r.stdout, r.stdout


def test_front_stage_arithmetic_is_bit_exact_with_cv2(hc):
    """SURVEY 8f-1: the product's BGR2GRAY and INTER_AREA per-sample functions (mc_math.cuh) and the tap/ROI
    builders (mc_tables.cpp), compiled for the CPU, against cv2 — integer-scale and fractional-scale paths."""
    rng = np.random.default_rng(5)
    px = rng.integers(0, 256, (200000, 3), dtype=np.uint8)
    g = np.empty(len(px), np.uint8)
    hc.hc_bgr2gray(px.ctypes.data_as(C.c_void_p), len(px), g.ctypes.data_as(C.c_void_p))
    assert np.array_equal(g, cv2.cvtColor(px[None], cv2.COLOR_BGR2GRAY)[0])
    for c in (1, 3):
        for (h, w, d) in ((50, 67, 2), (101, 77, 3), (37, 91, 4), (135, 241, 7), (64, 100, 8), (33, 35, 2), (90, 121, 5),
                          (48, 64, 2), (51, 69, 3), (64, 96, 4), (540, 960, 8), (270, 480, 5), (7, 9, 8), (216, 383, 2), (60, 60, 6)):
            dw, dh = max(1, w // d), max(1, h // d)
            src = rng.integers(0, 256, (h, w, c) if c > 1 else (h, w), dtype=np.uint8)
            ref = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_AREA)
            dst = np.empty_like(ref)
            hc.hc_resize_area(src.ctypes.data_as(C.c_void_p), h, w, c, dw, dh, dst.ctypes.data_as(C.c_void_p))
            assert np.array_equal(dst, ref), (c, h, w, d)
    out = (C.c_int * 4)()
    for (cols, rows, rx, ry, rw, rh) in ((1920, 1080, 0.25, 0.25, 0.5, 0.5), (640, 480, 0.1, 0.9, 0.95, 0.5), (333, 77, 0.0, 0.0, 1.0, 1.0),
                                          (100, 100, 0.995, 0.5, 0.2, 0.001), (1919, 1079, 0.3333, 0.6667, 0.3333, 0.25)):
        hc.hc_roi(cols, rows, 1, C.c_float(rx), C.c_float(ry), C.c_float(rw), C.c_float(rh), out)
        cfg = O.ProcessorConfig(preprocess=O.PreprocessParams(1, True, rx, ry, rw, rh))
        img = np.zeros((rows, cols), np.uint8)
        _, cropped = O.preprocess(img, cfg)
        assert (out[2], out[3]) == (cropped.shape[1], cropped.shape[0]), (cols, rows, list(out))


def test_c_abi_is_an_exception_firewall(built):
    """include/magcore_b200.h: "no exceptions cross this boundary".  The test hook mc_debug_inject_exception(n) makes
    the n-th guarded entry on this thread throw std::bad_alloc from INSIDE the body; the call must come back with
    MC_ERR_INTERNAL and a message (not std::terminate the process), and the library must keep working afterwards.
    (Error convention of the chain above the adapter: reference src/processing/ProcessingChain.cpp:50-62.)"""
    lib = capi.lib()
    raw = C.CDLL(built[0])
    raw.mc_debug_inject_exception.argtypes = [C.c_int]
    raw.mc_debug_inject_exception.restype = None
    a, b = (C.c_double * 3)(), (C.c_double * 3)()
    raw.mc_debug_inject_exception(1)
    assert lib.mc_butterworth(2, 0.2, a, b) == capi.MC_ERR_INTERNAL
    assert b"bad_alloc" in lib.mc_last_error(None)
    assert lib.mc_butterworth(2, 0.2, a, b) == capi.MC_OK and abs(a[0] - 1.0) < 1e-15     # disarmed, still works
    p = capi.McParams()
    lib.mc_params_from_ui(C.byref(p), 0, 20, 50.0, 0.4, 3.0, 0, 4, 30.0)
    g = (C.c_float * 5)()
    raw.mc_debug_inject_exception(2)                                                       # the SECOND entry throws
    assert lib.mc_motion_gains(C.byref(p), 4, 640, 480, g) == capi.MC_OK
    assert lib.mc_motion_gains(C.byref(p), 4, 640, 480, g) == capi.MC_ERR_INTERNAL
    assert lib.mc_motion_gains(C.byref(p), 4, 640, 480, g) == capi.MC_OK
    # a throw inside mc_create_lanes must not leak through either (no device here: the NO_DEVICE return comes first,
    # on a GPU box the injected throw is caught)
    h = C.c_void_p()
    raw.mc_debug_inject_exception(1)
    st = lib.mc_create_lanes(0, 1, C.byref(h))
    assert st in (capi.MC_ERR_NO_DEVICE, capi.MC_ERR_INTERNAL) and not h.value
    raw.mc_debug_inject_exception(0)
    # argument validation added with it: lane count bounds (grid.z = lanes * channels)
    assert lib.mc_create_lanes(0, 0, C.byref(h)) == capi.MC_ERR_INVALID
    assert lib.mc_create_lanes(0, capi.MC_MAX_LANES + 1, C.byref(h)) == capi.MC_ERR_INVALID


def test_sass_of_the_built_library_has_the_claimed_instructions():
    """cuobjdump works without a GPU: the fused level kernels use TMA (UTMALDG + mbarrier SYNCS, three bulk copies with
    the state prefetch), each ingest LUT gather is one 128-bit + one 64-bit load, the strip egress prefetches into L1
    and has no barrier, and the
    Phase egress clips NaN with an explicit select — ptxas folded fmaxf/fminf into FFMA.SAT (NaN -> 0) in round 1, which
    the CPU emulation cannot see (tools/check_sass.py)."""
    import shutil
    import subprocess
    import sys
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not installed")
    import __graft_entry__ as g
    if not os.path.exists(os.path.join(g.PKG, "libmagcore_b200.so")):
        g.build()
    r = subprocess.run([sys.executable, os.path.join(g.ROOT, "tools", "check_sass.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:]
