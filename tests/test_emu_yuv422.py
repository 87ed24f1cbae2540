"""Packed 4:2:2 camera frames into the chain on the CUDA-on-CPU emulation (tests/cuda_emu) at small sizes: the checkers of
test_gpu_yuv422.py, so the front's 32-bit and byte group reads, the always-written frames, the compose pane kind and the
host call are checked without a GPU.  They run again with asynchronous streams in a random order."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
from test_gpu_chain_lanes import MODES
from test_gpu_yuv422 import check_compose_yuv, check_yuv

pytestmark = pytest.mark.emu

W, H = 46, 29


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("order", [capi.MC_YUV422_YUYV, capi.MC_YUV422_UYVY], ids=["yuyv", "uyvy"])
@pytest.mark.parametrize("lay_kw", [dict(pitch=2 * W + 4), dict(pitch=2 * W + 3, lane_rows=1, offset=1)], ids=["vec", "bytes"])
def test_front_on_emulation(emu, order, lay_kw):
    steps = [("clip", 2), ("cfg", dict(down=3, roi=(0.03, 0.1, 0.8, 0.85), gray=True)), ("frame",),
             ("cfg", dict(gray=True)), ("frame",)]
    check_yuv(O.MODE_NONE, MODES["laplace"][1], W, H, steps, lanes=2, order=order, lay_kw=lay_kw, pads=(1, 2))


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_chain_lanes_on_emulation(emu, mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("clip", 2), ("restart", 1), ("hold", 2, 1), ("frame",), ("bgr",), ("hold", 2, 0),
             ("cfg", dict(down=2)), ("nv12",), ("clip", 2)]
    check_yuv(mode, ui, W, H + 1, steps, lanes=3, order=capi.MC_YUV422_UYVY)


def test_color_on_emulation(emu):
    mode, ui = MODES["color"]
    check_yuv(mode, ui, W, H, [("frame",), ("clip", 3), ("cfg", dict(gray=True)), ("frame",)], want_orig=False)


@pytest.mark.parametrize("split", [capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM])
@pytest.mark.parametrize("fmt,gray", [(capi.MC_CANVAS_BGR, True), (capi.MC_CANVAS_NV12, False)])
def test_compose_on_emulation(emu, split, fmt, gray):
    steps = [("frame",), ("cfg", dict(roi=(0.1, 0.15, 0.7, 0.8))), ("clip", 2), ("cfg", dict(down=2)), ("frame",)]
    check_compose_yuv(O.MODE_LAPLACE, MODES["laplace"][1], 64, 30, fmt, split, steps, lanes=2, gray=gray, pad=5, lane_rows=1,
                      uv_gap=3)
    check_compose_yuv(O.MODE_LAPLACE, MODES["laplace"][1], W, H, fmt, split, steps[:2] + [("frame",)], gray=gray,
                      order=capi.MC_YUV422_UYVY, lay_kw=dict(pitch=2 * W + 2, offset=2))


def test_with_asynchronous_random_streams():
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "11"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
