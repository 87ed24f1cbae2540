"""Moving a lane's temporal state (mc_save_lane / mc_load_lane) on the CUDA-on-CPU emulation (tests/cuda_emu): the
checks of test_gpu_lane_state.py without a GPU, and with asynchronous streams, where a save that did not wait for the
handle's stream would read planes the kernels have not written yet."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from test_gpu_lane_state import (check_blob_sizes, check_color, check_errors, check_laplace, check_laplace_unbounded,
                                 check_moves, check_phase)

pytestmark = pytest.mark.emu

W, H = 84, 46


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_laplace_lane_state_on_emulation(emu):
    check_laplace(W, H)
    check_laplace_unbounded(W, H)


def test_phase_lane_state_on_emulation(emu):
    check_phase(80, 60)


def test_color_lane_state_on_emulation(emu):
    check_color(32, 24, n_tail=6)


def test_lane_moves_on_emulation(emu):
    check_moves(W, H)


def test_lane_state_errors_on_emulation(emu):
    check_errors(W, H)
    check_blob_sizes(W, H)


@pytest.mark.parametrize("seed", ["3", "11"])
def test_lane_state_with_asynchronous_random_streams(seed):
    """The moves in a fresh process (the emulation reads CUDA_EMU_ASYNC once per process): every stream's work runs
    later, in a random order across streams, so the save's copies must be ordered on the handle's stream and waited for."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "laplace_lane_state_on or lane_moves_on"], env=env, capture_output=True,
                       text=True, timeout=2400)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
