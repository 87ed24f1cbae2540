"""The facts the planar 4:2:0 paths rest on, without a GPU: cv2 converts I420 and YV12 with the arithmetic of its NV12
conversion on every (Y, Cb, Cr) triple, YV12 is I420 with its chroma planes swapped, an NV12 canvas de-interleaved is
cv2's BGR2YUV_I420 of the BGR canvas; and the ctypes binding of mc_yuv420p, mc_canvas and the new entry points matches
include/magcore_b200.h."""
import ctypes as C
import os
import re
import subprocess

import cv2
import numpy as np

from lvm_b200 import capi
from compose_oracle import compose
from test_gpu_nv12 import to_nv12

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "magcore_b200.h")


def every_triple(w=4096):
    """-> (Y [w][w], Cb [w/2][w/2], Cr [w/2][w/2]): 2x2 block b carries the pair (b >> 8 & 255, b & 255) of b % 2^16 and
    the lumas 4r .. 4r + 3 of r = b >> 16, so every (Y, Cb, Cr) triple occurs once"""
    b = np.arange((w // 2) ** 2, dtype=np.uint32).reshape(w // 2, w // 2)
    pair, r = b & 0xFFFF, (b >> 16) & 63
    y = np.empty((w, w), np.uint8)
    for dy in (0, 1):
        for dx in (0, 1):
            y[dy::2, dx::2] = 4 * r + 2 * dy + dx
    return y, (pair >> 8).astype(np.uint8), (pair & 255).astype(np.uint8)


def test_i420_and_yv12_equal_nv12_on_every_triple():
    y, u, v = every_triple()
    w = y.shape[1]
    nv12 = np.concatenate([y, np.stack([u, v], -1).reshape(-1, w)])
    i420 = np.concatenate([y.ravel(), u.ravel(), v.ravel()]).reshape(-1, w)
    yv12 = np.concatenate([y.ravel(), v.ravel(), u.ravel()]).reshape(-1, w)
    want = cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12)
    assert np.array_equal(cv2.cvtColor(i420, cv2.COLOR_YUV2BGR_I420), want)
    assert np.array_equal(cv2.cvtColor(yv12, cv2.COLOR_YUV2BGR_YV12), want)


def test_bgr2yuv_yv12_is_i420_with_the_chroma_planes_swapped():
    for h, w in [(2, 2), (30, 46), (78, 134)]:
        bgr = np.random.default_rng(w).integers(0, 256, (h, w, 3), dtype=np.uint8)
        i420, yv12 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420).ravel(), cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_YV12).ravel()
        n, q = w * h, w * h // 4
        assert np.array_equal(yv12[:n], i420[:n])
        assert np.array_equal(yv12[n:n + q], i420[n + q:]) and np.array_equal(yv12[n + q:], i420[n:n + q])


def test_nv12_canvas_deinterleaved_is_bgr2yuv_i420():
    rng = np.random.default_rng(5)
    for split in (capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM):
        original = rng.integers(0, 256, (31, 45, 3), dtype=np.uint8)
        cur = rng.integers(0, 256, (31, 45), dtype=np.uint8)   # a gray pane, expanded as GRAY2BGR
        canvas = compose(original, cur, split)
        h, w = canvas.shape[:2]
        nv = to_nv12(canvas)
        uv = nv[h:]
        planar = np.concatenate([nv[:h].ravel(), uv[:, 0::2].ravel(), uv[:, 1::2].ravel()])
        assert np.array_equal(planar, cv2.cvtColor(canvas, cv2.COLOR_BGR2YUV_I420).ravel()), split


def test_binding_matches_the_header(tmp_path):
    """the four entry points are declared and bound; McYuv420p and McCanvas have the C layout (offsets and sizes printed
    by a C program compiled against the header); MC_CANVAS_I420 is 2"""
    text = open(HEADER).read()
    names = ("mc_chain_process_yuv420p_device", "mc_chain_compose_yuv420p_device", "mc_chain_submit_yuv420p",
             "mc_chain_compose_submit_yuv420p")
    for n in names:
        assert re.search(r"\bmc_status\s+" + n + r"\s*\(", text), n
        assert n in capi.SIGNATURES and capi.SIGNATURES[n][1][1]._type_ is capi.McYuv420p, n
    assert re.search(r"MC_CANVAS_I420\s*=\s*2\b", text) and capi.MC_CANVAS_I420 == 2
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "magcore_b200.h"\n'
                   '#define F(s, f) printf("%s.%s %zu\\n", #s, #f, offsetof(s, f));\n'
                   "int main(void) {\n"
                   "F(mc_yuv420p, y) F(mc_yuv420p, u) F(mc_yuv420p, v) F(mc_yuv420p, pitch) F(mc_yuv420p, chroma_pitch)\n"
                   "F(mc_yuv420p, lane_stride)\n"
                   "F(mc_canvas, format) F(mc_canvas, data) F(mc_canvas, uv) F(mc_canvas, pitch) F(mc_canvas, lane_stride)\n"
                   'printf("mc_yuv420p %zu\\nmc_canvas %zu\\n", sizeof(mc_yuv420p), sizeof(mc_canvas));\n'
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for cname, cls in (("mc_yuv420p", capi.McYuv420p), ("mc_canvas", capi.McCanvas)):
        assert int(got[cname]) == C.sizeof(cls), cname
        for field, _ in cls._fields_:
            assert int(got[f"{cname}.{field}"]) == getattr(cls, field).offset, (cname, field)
