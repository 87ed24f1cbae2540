"""Planar 4:2:0 frames (I420 / YV12) and I420 canvases on the CUDA-on-CPU emulation (tests/cuda_emu) at small sizes: the
checkers of test_gpu_yuv420p.py, so the front's planar chroma reads, the compose kernel's I420 pane reads and chroma
stores (vector and byte paths), the three-plane staging and copies of the submits and the error paths are checked
without a GPU.  They run again with asynchronous streams in a random order."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
import test_gpu_chain_submit as chain_submit
import test_gpu_compose_submit as compose_submit
from test_gpu_chain_lanes import MODES
from test_gpu_yuv420p import (BGR, I420, LR, NONE, NV12, TB, Canvas420, ChainSource, ClipSource, check_420, check_compose_420,
                              test_errors_return_before_any_launch_or_copy as check_errors)

pytestmark = pytest.mark.emu

W, H = 46, 30
VEC = dict(pitch=W + 10, chroma_pitch=W // 2 + 9, arrangement="uvy")            # 8-byte luma rows, 4-byte chroma rows
BYTES = dict(pitch=W + 2, chroma_pitch=W // 2 + 1, arrangement="far", offset=1, gap=1)


@pytest.fixture()
def emu(monkeypatch):
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    monkeypatch.setattr(chain_submit, "Source", ChainSource)
    monkeypatch.setattr(compose_submit, "ClipSource", ClipSource)
    monkeypatch.setattr(compose_submit, "Canvas", Canvas420)
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("lay_kw", [VEC, BYTES], ids=["vec", "bytes"])
def test_front_on_emulation(emu, lay_kw):
    steps = [("clip", 2), ("cfg", dict(down=3, roi=(0.03, 0.1, 0.8, 0.85), gray=True)), ("frame",),
             ("cfg", dict(roi=(0.015, 0.03, 0.6, 0.8))), ("frame",), ("cfg", dict(down=2)), ("frame",)]
    check_420(O.MODE_NONE, MODES["laplace"][1], W, H, steps, lanes=2, lay_kw=lay_kw)


@pytest.mark.parametrize("mname", list(MODES))
def test_chain_lanes_on_emulation(emu, mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("clip", 2), ("restart", 1), ("hold", 2, 1), ("frame",), ("bgr",), ("hold", 2, 0), ("lp", 0),
             ("cfg", dict(down=2)), ("nv12",), ("yuyv",), ("clip", 2)]
    check_420(mode, ui, W, H, steps, lanes=3, lay_kw=VEC, color_lifecycle=mname == "color")


@pytest.mark.parametrize("split", [NONE, LR, TB], ids=["none", "left_right", "top_bottom"])
@pytest.mark.parametrize("fmt", [BGR, NV12, I420], ids=["bgr_canvas", "nv12_canvas", "i420_canvas"])
@pytest.mark.parametrize("lay_kw", [VEC, BYTES], ids=["vec", "bytes"])
def test_compose_on_emulation(emu, split, fmt, lay_kw):
    steps = [("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 2), ("hold", 1, 1), ("frame",), ("hold", 1, 0)]
    aligned = lay_kw is VEC
    check_compose_420(O.MODE_LAPLACE, MODES["laplace"][1], 64 if aligned else W, 32 if aligned else H, fmt, split, steps,
                      lanes=2, labels=True, lay_kw=dict(pitch=64, chroma_pitch=32, arrangement="uvy") if aligned else lay_kw,
                      pad=0 if aligned else 6, lane_rows=0 if aligned else 1,
                      uv_gap=0 if aligned else 3)


@pytest.mark.parametrize("src", ["bgr", "gray", "nv12", "yuyv"])
def test_i420_canvas_from_other_sources_on_emulation(emu, src):
    check_compose_420(O.MODE_LAPLACE, MODES["laplace"][1], W, H, I420, LR, [("frame",), ("clip", 2)], src=src, labels=True, pad=4)


@pytest.mark.parametrize("kind,fmt,depth", [("i420", I420, 3), ("i420", BGR, 1), ("nv12", I420, 5)])
def test_submits_on_emulation(emu, kind, fmt, depth):
    compose_submit.check_compose_submit(kind, "roi", "laplace", lanes=2, depth=depth, clips=(4, 3, 1, 4, 2), fmt=fmt, split=LR,
                                        w=W, h=H)
    if kind == "i420":
        chain_submit.check_chain_submit("i420", "down2", "laplace", lanes=2, depth=depth, n=8, w=W, h=H)


def test_errors_on_emulation(emu):
    check_errors()


def test_with_asynchronous_random_streams():
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "13"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
