"""The pipelined export canvas from host clips (mc_chain_compose_submit / _nv12 / _yuv422, collected by mc_collect) on the
CUDA-on-CPU emulation (tests/cuda_emu): the checkers of test_gpu_compose_submit at a small size, equal to a twin handle's
device compose calls bit for bit.  The same checks run again with asynchronous streams in a random order.  There a
canvas written to handle scratch instead of the slot's own output, a slot reused before its download finished, or an
upload, download or staging copy that is not ordered by a stream or an event wait gives wrong bytes."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from test_gpu_compose_submit import BGR, LR, NONE, NV12, TB, check_compose_submit, check_errors, check_interleaved

pytestmark = pytest.mark.emu

W, H = 66, 38


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("kind,front,fmt,split,pins", [
    ("bgr", "roi", BGR, LR, ((False, False), (True, True))), ("gray", "down2", NV12, TB, ((True, False),)),
    ("nv12", "gray", NV12, LR, ((False, True), (True, False))), ("yuyv", "none", BGR, NONE, ((True, True),)),
    ("uyvy", "roi", NV12, NONE, ((False, False),))])
def test_compose_submit_on_emulation(emu, kind, front, fmt, split, pins):
    check_compose_submit(kind, front, "laplace", lanes=1, depth=3, fmt=fmt, split=split, pins=pins, w=W, h=H)


@pytest.mark.parametrize("mname,depth", [("laplace", 5), ("phase", 3), ("color", 1)])
def test_compose_submit_lanes_on_emulation(emu, mname, depth):
    check_compose_submit("nv12", "down2", mname, lanes=3, depth=depth, clips=(6, 3, 1, 6, 3, 1, 6, 2), fmt=BGR, split=LR,
                         w=W, h=H)


def test_compose_submit_fifo_on_emulation(emu):
    check_interleaved(W, H, pinned=True)


def test_compose_submit_errors_on_emulation(emu):
    check_errors(W, H)


@pytest.mark.parametrize("seed", ["3", "11"])
def test_compose_submit_with_asynchronous_random_streams(seed):
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
