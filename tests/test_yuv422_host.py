"""The packed 4:2:2 conversion's per-pixel function (yuv422_to_bgr_px in csrc/mc_math.cuh), compiled for the CPU from
tests/hostcheck/yuv422check.cpp, against cv2's COLOR_YUV2BGR_YUYV / _UYVY for all 2^24 (Y, Cb, Cr) triples in both byte
orders, and on random frames with padded rows and odd heights."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODES = {0: cv2.COLOR_YUV2BGR_YUYV, 1: cv2.COLOR_YUV2BGR_UYVY}


@pytest.fixture(scope="module")
def hc(tmp_path_factory):
    """tests/hostcheck/yuv422check.cpp built with the flags of the product's host build (no FMA contraction)"""
    lib = str(tmp_path_factory.mktemp("yuv422check") / "libyuv422check.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", "/usr/local/cuda/include", "-I",
                    os.path.join(ROOT, "live-video-magnification_b200", "csrc"),
                    os.path.join(ROOT, "tests", "hostcheck", "yuv422check.cpp"), "-o", lib], check=True)
    return C.CDLL(lib)


def every_triple(order, w=4096):
    """-> a packed 4:2:2 frame [h][2w] of that byte order (h = 2^23 / (w / 2) rows) holding every (Y, Cb, Cr) triple once:
    group i carries the pair (Cb, Cr) = (i >> 8 & 255, i & 255) and the luma values 2 (i >> 16) and 2 (i >> 16) + 1"""
    i = np.arange(1 << 23, dtype=np.uint32)
    y0, u, v = (i >> 16) * 2, (i >> 8) & 255, i & 255
    grp = np.stack([y0, u, y0 + 1, v] if order == 0 else [u, y0, v, y0 + 1], -1).astype(np.uint8)
    return grp.reshape(-1, 2 * w)


def hc_convert(hc, frame, w, h, order, pitch=None):
    out = np.empty((h, w, 3), np.uint8)
    hc.yc_yuv422_to_bgr(frame.ctypes.data_as(C.c_void_p), C.c_size_t(pitch or 2 * w), w, h, order,
                        out.ctypes.data_as(C.c_void_p))
    return out


@pytest.mark.parametrize("order", [0, 1], ids=["yuyv", "uyvy"])
def test_every_triple_equals_cv2(hc, order):
    x = every_triple(order)
    h, w = x.shape[0], x.shape[1] // 2
    assert np.array_equal(hc_convert(hc, x, w, h, order), cv2.cvtColor(x.reshape(h, w, 2), CODES[order]))


def test_both_orders_of_the_same_bytes_agree():
    """swapping each byte pair turns YUYV into UYVY: cv2 gives the same BGR (what the device paths rely on)"""
    x = np.random.default_rng(1).integers(0, 256, (33, 2 * 86), dtype=np.uint8)
    swapped = x.reshape(33, -1, 2)[..., ::-1].reshape(33, -1).copy()
    assert np.array_equal(cv2.cvtColor(x.reshape(33, 86, 2), CODES[0]), cv2.cvtColor(swapped.reshape(33, 86, 2), CODES[1]))


@pytest.mark.parametrize("w,h,pad", [(2, 1, 0), (6, 3, 2), (34, 9, 1), (130, 67, 64)])
@pytest.mark.parametrize("order", [0, 1], ids=["yuyv", "uyvy"])
def test_random_frames_with_padded_rows(hc, w, h, pad, order):
    rng = np.random.default_rng(w + pad)
    buf = rng.integers(0, 256, (h, 2 * w + pad), dtype=np.uint8)
    want = cv2.cvtColor(np.ascontiguousarray(buf[:, :2 * w]).reshape(h, w, 2), CODES[order])
    assert np.array_equal(hc_convert(hc, buf, w, h, order, 2 * w + pad), want)
