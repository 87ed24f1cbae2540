"""RGB frames and RGB canvases on the CUDA-on-CPU emulation (tests/cuda_emu) at small sizes: the checkers of
test_gpu_rgb.py, so the front's channel-base reads of every layout, the compose kernel's RGB and planar RGB stores (vector
and byte paths), the staging and copies of packed and planar submits and the error paths are checked without a GPU.  They
run again with asynchronous streams in a random order."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
import test_gpu_chain_submit as chain_submit
import test_gpu_compose_submit as compose_submit
import test_gpu_yuv422 as yuv422
from test_gpu_chain_lanes import MODES
from test_gpu_rgb import (BGR_C, BPP, BGRA, I420_C, LR, NONE, PLANAR, PLANAR_C, RGB, RGB_C, RGBA, TB, CanvasRgb, ChainSource,
                          ClipSource, Rgb, check_compose_rgb, check_rgb_twins, convert, from_bgr, rgb_device_call,
                          test_errors_return_before_any_launch_or_copy as check_errors)

pytestmark = pytest.mark.emu

W, H = 46, 30


@pytest.fixture()
def emu(monkeypatch):
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    monkeypatch.setattr(chain_submit, "Source", ChainSource)
    monkeypatch.setattr(compose_submit, "ClipSource", ClipSource)
    monkeypatch.setattr(compose_submit, "Canvas", CanvasRgb)
    monkeypatch.setattr(yuv422, "from_bgr", from_bgr)
    monkeypatch.setattr(yuv422, "convert", convert)
    monkeypatch.setattr(yuv422, "Yuv", Rgb)
    monkeypatch.setattr(yuv422, "yuv_device_call", rgb_device_call)
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("layout", [RGB, RGBA, BGRA, PLANAR], ids=["rgb", "rgba", "bgra", "planar"])
def test_front_on_emulation(emu, layout):
    steps = [("clip", 2), ("cfg", dict(down=3, roi=(0.03, 0.1, 0.8, 0.85), gray=True)), ("frame",),
             ("cfg", dict(roi=(0.015, 0.03, 0.6, 0.8))), ("frame",), ("cfg", dict(down=2)), ("frame",)]
    yuv422.check_yuv(O.MODE_NONE, MODES["laplace"][1], W, H, steps, lanes=2, order=layout,
                     lay_kw=dict(pitch=W * BPP[layout] + 3, offset=1, arrangement="far", gap=1))


@pytest.mark.parametrize("mname", list(MODES))
def test_chain_lanes_on_emulation(emu, mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("clip", 2), ("restart", 1), ("hold", 2, 1), ("frame",), ("bgr",), ("hold", 2, 0), ("lp", 0),
             ("cfg", dict(down=2)), ("nv12",), ("yuyv",), ("i420",), ("clip", 2)]
    check_rgb_twins(mode, ui, steps, lanes=3, layout=PLANAR, w=W, h=H)


@pytest.mark.parametrize("split", [NONE, LR, TB], ids=["none", "left_right", "top_bottom"])
@pytest.mark.parametrize("fmt", [BGR_C, I420_C, RGB_C, PLANAR_C], ids=["bgr_canvas", "i420_canvas", "rgb_canvas", "planar_canvas"])
@pytest.mark.parametrize("aligned", [True, False], ids=["vec", "bytes"])
def test_compose_on_emulation(emu, split, fmt, aligned):
    steps = [("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 2), ("hold", 1, 1), ("frame",), ("hold", 1, 0)]
    layout = PLANAR if aligned else RGBA
    check_compose_rgb(O.MODE_LAPLACE, MODES["laplace"][1], 64 if aligned else W, 32 if aligned else H, fmt, split, steps,
                      lanes=2, layout=layout, labels=True,
                      lay_kw=None if aligned else dict(pitch=4 * W + 3, offset=1), pad=0 if aligned else 6,
                      lane_rows=0 if aligned else 1)


@pytest.mark.parametrize("src", ["bgr", "gray", "nv12", "yuyv", "i420"])
def test_rgb_canvases_from_other_sources_on_emulation(emu, src):
    for fmt in (RGB_C, PLANAR_C):
        check_compose_rgb(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, LR, [("frame",), ("clip", 2)], src=src, labels=True,
                          pad=4)


@pytest.mark.parametrize("kind,fmt,depth", [("planar", PLANAR_C, 3), ("rgb", RGB_C, 1), ("bgra", BGR_C, 5), ("nv12", PLANAR_C, 3)])
def test_submits_on_emulation(emu, kind, fmt, depth):
    compose_submit.check_compose_submit(kind, "roi", "laplace", lanes=2, depth=depth, clips=(4, 3, 1, 4, 2), fmt=fmt, split=LR,
                                        w=W, h=H)
    if kind != "nv12":
        chain_submit.check_chain_submit(kind, "down2", "laplace", lanes=2, depth=depth, n=8, w=W, h=H)


def test_errors_on_emulation(emu):
    check_errors()


def test_with_asynchronous_random_streams():
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "13"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
