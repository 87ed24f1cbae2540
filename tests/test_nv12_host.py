"""The NV12 conversions' per-pixel functions (nv12_to_bgr_px / bgr_to_ycc_px in csrc/mc_math.cuh), compiled for the CPU
from tests/hostcheck/nv12check.cpp, against cv2 on every input: all 2^24 (Y, Cb, Cr) triples and all 2^24 BGR colours."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

_u8p = C.POINTER(C.c_uint8)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hc(tmp_path_factory):
    """tests/hostcheck/nv12check.cpp built with the flags of the product's host build (no FMA contraction)"""
    lib = str(tmp_path_factory.mktemp("nv12check") / "libnv12check.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I",
                    os.path.join(ROOT, "live-video-magnification_b200", "csrc"),
                    os.path.join(ROOT, "tests", "hostcheck", "nv12check.cpp"), "-o", lib], check=True)
    return C.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(_u8p)


def hc_nv12_to_bgr(hc, y, u, v):
    y, u, v = (np.ascontiguousarray(a, np.uint8) for a in (y, u, v))
    out = np.empty(y.shape + (3,), np.uint8)
    hc.nc_nv12_to_bgr(_p(y), _p(u), _p(v), y.size, _p(out))
    return out


def hc_bgr_to_ycc(hc, bgr):
    bgr = np.ascontiguousarray(bgr, np.uint8)
    out = np.empty(bgr.shape, np.uint8)
    hc.nc_bgr_to_ycc(_p(bgr), bgr.size // 3, _p(out))
    return out


def i420_chroma(i420, w, h):
    """The Cb and Cr planes ([h/2][w/2]) of cv2's I420 output."""
    flat, n = i420.ravel(), w * h
    return flat[n:n + n // 4].reshape(h // 2, w // 2), flat[n + n // 4:].reshape(h // 2, w // 2)


def all_yuv_frames(width=4096):
    """Yields (nv12 [3h/2][w], Y [h][w], U, V full resolution): every (Y, Cb, Cr) once over the 64 frames.  Each 2x2
    block carries one (Cb, Cr) pair; its four pixels take four consecutive luma values."""
    u, v = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    bw = width // 2
    bh = 65536 // bw
    uv = np.stack([u.reshape(bh, bw), v.reshape(bh, bw)], -1).reshape(bh, width).astype(np.uint8)
    uf = np.repeat(np.repeat(u.reshape(bh, bw), 2, 0), 2, 1).astype(np.uint8)
    vf = np.repeat(np.repeat(v.reshape(bh, bw), 2, 0), 2, 1).astype(np.uint8)
    for y0 in range(0, 256, 4):
        y = np.broadcast_to(np.arange(y0, y0 + 4, dtype=np.uint8).reshape(1, 2, 1, 2), (bh, 2, bw, 2)).reshape(2 * bh, width)
        yield np.concatenate([y, uv], 0), y, uf, vf


def all_bgr_blocks(part, rng):
    """4 parts of 2^22 colours: each colour is the top-left pixel of a 2x2 block whose other three pixels are random."""
    cols = np.arange(part << 22, (part + 1) << 22, dtype=np.uint32)
    tl = np.stack([cols & 255, (cols >> 8) & 255, cols >> 16], -1).astype(np.uint8).reshape(1024, 4096, 3)
    img = rng.integers(0, 256, (2048, 8192, 3), dtype=np.uint8)
    img[::2, ::2] = tl
    return img, tl


def test_nv12_to_bgr_equals_cv2_for_every_yuv(hc):
    for nv, y, u, v in all_yuv_frames():
        assert np.array_equal(hc_nv12_to_bgr(hc, y, u, v), cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12))


def test_bgr_to_ycc_equals_cv2_for_every_colour(hc):
    rng = np.random.default_rng(7)
    for part in range(4):
        img, tl = all_bgr_blocks(part, rng)
        h, w = img.shape[:2]
        i420 = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)
        ycc = hc_bgr_to_ycc(hc, img)
        assert np.array_equal(ycc[..., 0], i420[:h])
        cb, cr = i420_chroma(i420, w, h)
        assert np.array_equal(ycc[::2, ::2, 1], cb) and np.array_equal(ycc[::2, ::2, 2], cr)
        assert np.array_equal(hc_bgr_to_ycc(hc, tl)[..., 1:], np.stack([cb, cr], -1))


@pytest.mark.parametrize("w,h", [(2, 2), (6, 4), (34, 10), (130, 66)])
def test_small_widths_equal_cv2(hc, w, h):
    rng = np.random.default_rng(w)
    nv = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    uv = nv[h:].reshape(h // 2, w // 2, 2)
    up = lambda a: np.repeat(np.repeat(a, 2, 0), 2, 1)
    assert np.array_equal(hc_nv12_to_bgr(hc, nv[:h], up(uv[..., 0]), up(uv[..., 1])), cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12))
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    i420 = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)
    ycc = hc_bgr_to_ycc(hc, img)
    assert np.array_equal(ycc[..., 0], i420[:h])
    cb, cr = i420_chroma(i420, w, h)
    assert np.array_equal(ycc[::2, ::2, 1], cb) and np.array_equal(ycc[::2, ::2, 2], cr)
