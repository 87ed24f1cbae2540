"""Per-lane parameters (mc_set_lane_params) on the CUDA-on-CPU emulation (tests/cuda_emu): the per-lane table of the
Laplace kernels, checked bit for bit against 1-lane handles without a GPU, and the table upload's stream order against
frames in flight (asynchronous streams)."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from test_gpu_lane_params import (check_color, check_color_refusal, check_equal_override_is_none, check_errors,
                                  check_laplace_matrix, check_phase, check_schedule)

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_laplace_lane_params_on_emulation(emu):
    check_laplace_matrix(83, 45)
    check_equal_override_is_none(83, 45)
    check_errors()


@pytest.mark.parametrize("entry,clip,depth", [("frame", 1, 3), ("clip", 1, 3), ("clip", 7, 3), ("submit", 1, 1), ("submit", 1, 5)])
def test_lane_param_schedules_on_emulation(emu, entry, clip, depth):
    check_schedule(83, 45, entry, clip, depth)


@pytest.mark.parametrize("entry,clip", [("frame", 1), ("clip", 3)])
def test_phase_lane_params_on_emulation(emu, entry, clip):
    check_phase(80, 60, entry, clip)


def test_color_lane_params_on_emulation(emu):
    check_color(48, 32, n=36)
    check_color_refusal(48, 32)


@pytest.mark.parametrize("seed", ["3", "11"])
def test_lane_param_submits_with_asynchronous_random_streams(seed):
    """The submit schedules in a fresh process (the emulation reads CUDA_EMU_ASYNC once per process): the table upload
    must be ordered on the handle's stream against the frames in flight."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "schedules_on_emulation and submit"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
