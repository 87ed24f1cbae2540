"""Per-lane ROIs (mc_set_lane_roi) on the CUDA-on-CPU emulation (tests/cuda_emu) at small sizes: the checkers of
test_gpu_lane_roi.py, so the front's per-lane origins on every source, the per-lane structural restarts in all three
modes, the size check, resets, clears and lane blobs are checked against 1-lane twins without a GPU.  The submits run
again with asynchronous streams in a random order: the origins' upload must be ordered on the handle's stream against
the frames in flight."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from test_gpu_lane_roi import (SOURCES, check_clips, check_color_refusal, check_compose, check_downscale, check_errors,
                               check_magnifier_only, check_modes, check_reset_and_clear, check_save_load, check_sources,
                               check_submits, check_unequal_sizes)

pytestmark = pytest.mark.emu

W, H = 48, 32


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("kind", SOURCES)
def test_every_source_on_emulation(emu, kind):
    check_sources(kind, W, H)


@pytest.mark.parametrize("mname", ["laplace", "phase", "color"])
def test_modes_on_emulation(emu, mname):
    check_modes(mname, W, H)


def test_lane_rules_on_emulation(emu):
    check_color_refusal(W, H)
    check_unequal_sizes(W, H)
    check_reset_and_clear(W, H)
    check_save_load(W, H)
    check_magnifier_only(W, H)
    check_errors()


@pytest.mark.parametrize("down", [2, 3])
def test_downscale_on_emulation(emu, down):
    check_downscale(down, W, H)


def test_clips_and_compose_on_emulation(emu):
    check_clips(3, W, H)
    check_compose("bgr", capi.MC_CANVAS_BGR, W, H)
    check_compose("nv12", capi.MC_CANVAS_I420, W, H)


@pytest.mark.parametrize("depth", [1, 3])
def test_submits_on_emulation(emu, depth):
    check_submits(depth, W, H)


@pytest.mark.parametrize("seed", ["5", "17"])
def test_submits_with_asynchronous_random_streams(seed):
    """The submit checks in a fresh process (the emulation reads CUDA_EMU_ASYNC once per process)."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "submits_on_emulation or clips_and_compose"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
