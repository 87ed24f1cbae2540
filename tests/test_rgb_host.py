"""The facts the RGB paths rest on, without a GPU: cv2's RGB2BGR, RGBA2BGR and BGRA2BGR are byte permutations on every
colour whatever the alpha, a merge of the planes is the planar form, and BGR2RGB of a canvas is its byte swap; the ctypes
binding of mc_rgb, the canvas formats and the new entry points matches include/magcore_b200.h; and the kernels the RGB
paths run, k_compose and k_chain_front, compile without local-memory spills."""
import ctypes as C
import importlib.util
import os
import re
import subprocess

import cv2
import numpy as np

from lvm_b200 import capi
from compose_oracle import compose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "magcore_b200.h")


def every_colour():
    """-> 4096 x 4096 x 3 u8 BGR: every (B, G, R) triple once"""
    c = np.arange(1 << 24, dtype=np.uint32).reshape(4096, 4096)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8)


def test_rgb_layouts_to_bgr_are_byte_permutations_on_every_colour():
    bgr = every_colour()
    alpha = np.random.default_rng(1).integers(0, 256, bgr.shape[:2] + (1,), dtype=np.uint8)
    rgb = np.ascontiguousarray(bgr[..., ::-1])
    assert np.array_equal(cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR), bgr)
    assert np.array_equal(cv2.cvtColor(np.concatenate([rgb, alpha], -1), cv2.COLOR_RGBA2BGR), bgr)
    assert np.array_equal(cv2.cvtColor(np.concatenate([bgr, alpha], -1), cv2.COLOR_BGRA2BGR), bgr)
    r, g, b = (np.ascontiguousarray(rgb[..., k]) for k in range(3))   # a CHW tensor's planes
    assert np.array_equal(cv2.merge([b, g, r]), bgr)


def test_bgr2rgb_of_a_canvas_is_the_byte_swap():
    rng = np.random.default_rng(5)
    for split in (capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM):
        original = rng.integers(0, 256, (31, 45, 3), dtype=np.uint8)
        cur = rng.integers(0, 256, (31, 45), dtype=np.uint8)   # a gray pane, expanded as GRAY2BGR
        canvas = compose(original, cur, split)
        assert np.array_equal(cv2.cvtColor(canvas, cv2.COLOR_BGR2RGB), canvas[..., ::-1]), split
        planar = np.stack([canvas[..., 2], canvas[..., 1], canvas[..., 0]])   # one CHW tensor
        assert np.array_equal(planar.transpose(1, 2, 0), cv2.cvtColor(canvas, cv2.COLOR_BGR2RGB)), split


def test_binding_matches_the_header(tmp_path):
    """the four entry points are declared and bound; McRgb and McCanvas have the C layout (offsets and sizes printed by a
    C program compiled against the header); the layout and canvas constants are the header's"""
    text = open(HEADER).read()
    names = ("mc_chain_process_rgb_device", "mc_chain_compose_rgb_device", "mc_chain_submit_rgb", "mc_chain_compose_submit_rgb")
    for n in names:
        assert re.search(r"\bmc_status\s+" + n + r"\s*\(", text), n
        assert n in capi.SIGNATURES and capi.SIGNATURES[n][1][1]._type_ is capi.McRgb, n
    for name, value in (("MC_CANVAS_RGB", 3), ("MC_CANVAS_RGB_PLANAR", 4), ("MC_RGB_RGB", 0), ("MC_RGB_RGBA", 1),
                        ("MC_RGB_BGRA", 2), ("MC_RGB_PLANAR", 3)):
        assert re.search(name + r"\s*=\s*" + str(value) + r"\b", text) and getattr(capi, name) == value, name
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "magcore_b200.h"\n'
                   '#define F(s, f) printf("%s.%s %zu\\n", #s, #f, offsetof(s, f));\n'
                   "int main(void) {\n"
                   "F(mc_rgb, data) F(mc_rgb, g) F(mc_rgb, b) F(mc_rgb, pitch) F(mc_rgb, lane_stride) F(mc_rgb, layout)\n"
                   "F(mc_canvas, format) F(mc_canvas, data) F(mc_canvas, uv) F(mc_canvas, pitch) F(mc_canvas, lane_stride)\n"
                   'printf("mc_rgb %zu\\nmc_canvas %zu\\n", sizeof(mc_rgb), sizeof(mc_canvas));\n'
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for cname, cls in (("mc_rgb", capi.McRgb), ("mc_canvas", capi.McCanvas)):
        assert int(got[cname]) == C.sizeof(cls), cname
        for field, _ in cls._fields_:
            assert int(got[f"{cname}.{field}"]) == getattr(cls, field).offset, (cname, field)


def test_compose_and_front_do_not_spill():
    """every k_compose instance (BGR, 4:2:0, RGB and planar RGB canvases) and every k_chain_front instance (BGR with the
    RGB layouts, gray, 4:2:0, YUYV, UYVY) compiles without local-memory spills (the build's ptxas -v log)"""
    spec = importlib.util.spec_from_file_location("check_sass", os.path.join(ROOT, "tools", "check_sass.py"))
    sass = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sass)
    compose_ = sass.clip_spills("k_compose", "mc_preprocess")
    front = sass.clip_spills("k_chain_front", "mc_preprocess")
    assert len(compose_) == 4 and all(s == (0, 0) for s in compose_.values()), compose_
    assert len(front) == 5 and all(s == (0, 0) for s in front.values()), front
