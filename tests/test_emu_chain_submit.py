"""The pipelined host chain (mc_chain_submit / _nv12 / _yuv422, collected by mc_collect) on the CUDA-on-CPU emulation
(tests/cuda_emu): the checkers of test_gpu_chain_submit at a small size, equal to a twin handle's device chain calls bit
for bit.  The same checks run again with asynchronous streams in a random order.  There the chain's shared front scratch
(staging, held-lane flags, INTER_AREA tap tables) is reused by frames in flight across a ROI move and a hold, and an upload,
download or staging buffer that is not ordered by a stream or an event wait gives wrong bytes."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from test_gpu_chain_submit import check_chain_submit, check_errors, check_interleaved

pytestmark = pytest.mark.emu

W, H = 66, 38


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("kind,front,pins", [("bgr", "roi_down_gray", (False, False, False)), ("gray", "down3", (True, True, True)),
                                             ("nv12", "roi", (True, False, True)), ("yuyv", "down2", (False, True, False)),
                                             ("uyvy", "none", (True, True, False))])
def test_chain_submit_on_emulation(emu, kind, front, pins):
    check_chain_submit(kind, front, "laplace", lanes=2, depth=3, pins=pins, w=W, h=H)


@pytest.mark.parametrize("mname,depth", [("phase", 5), ("color", 1)])
def test_chain_submit_modes_on_emulation(emu, mname, depth):
    check_chain_submit("bgr", "roi_down_gray", mname, lanes=2, depth=depth, w=W, h=H)


def test_chain_submit_fifo_on_emulation(emu):
    check_interleaved(W, H, pinned=True)


def test_chain_submit_errors_on_emulation(emu):
    check_errors(W, H)


@pytest.mark.parametrize("seed", ["3", "11"])
def test_chain_submit_with_asynchronous_random_streams(seed):
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
