"""Color clips (mc_process_clip) on the CUDA-on-CPU emulation (tests/cuda_emu): the checkers of test_gpu_color_clip.py at
small sizes, so the per-virtual-lane table, the append slots, the per-frame windows and the taps after a clip are checked
bit for bit against frame calls without a GPU.  They run again with asynchronous streams in a random order."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
import test_gpu_color_clip as CC

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_warmup_and_a_clip_longer_than_the_window_on_emulation(emu):
    got = CC.check_color(35, 21, 3, [("clip", 5), ("clip", 14), ("clip", 21)], float_out=True)
    assert got[0][:, 0].tolist() == [0, 1, 1, 1, 1] and got[1].all() and got[2].all()


def test_gray_resize_and_framerate_changes_on_emulation(emu):
    CC.check_color(23, 19, 1, [("clip", 18), ("fps", 30.0), ("clip", 4), ("fps", 8.0), ("clip", 3), ("frames", 1),
                               ("fps", 7.0), ("clip", 5)], levels=1)


def test_lanes_of_different_lengths_on_emulation(emu):
    steps = [("clip", 4), ("restart", 1), ("hold", 2, 1), ("clip", 5), ("hold", 2, 0), ("clip", 3), ("restart", 0),
             ("clip", 6), ("reset",), ("clip", 2), ("none", 1), ("clip", 3)]
    CC.check_color(27, 17, 3, steps, lanes=3, options=CC.LIFECYCLE, float_out=True)


def test_chain_calls_on_emulation(emu):
    for kind in ("chain", "compose_nv12", "yuv422"):
        CC.check_chain_calls(kind, 40, 24, CC.CHAIN_STEPS)
    CC.check_chain_calls("chain", 40, 24, CC.CHAIN_STEPS, settings=dict(down=2, gray=True))


def test_launch_count_on_emulation(emu):
    CC.check_launches(35, 21, 2, 3)


@pytest.mark.parametrize("seed", ["5"])
def test_color_clip_with_asynchronous_random_streams(seed):
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
