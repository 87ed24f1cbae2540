"""Labels on the export canvas (mc_set_overlay) on the CUDA-on-CPU emulation (tests/cuda_emu) at small sizes: the small
cases of test_gpu_compose_labels.py, so the overlay's rect tests, index and palette reads and the mapped byte and 64-bit
paths are checked without a GPU.  They run again with asynchronous streams in a random order, where an overlay upload
that is not ordered on the handle's stream gives wrong canvases."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
import test_gpu_compose_labels as G

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("split", ["left_right", "top_bottom", "none"])
@pytest.mark.parametrize("src,fmt,gray", [("bgr", capi.MC_CANVAS_NV12, False), ("gray", capi.MC_CANVAS_BGR, False),
                                          ("nv12", capi.MC_CANVAS_NV12, True)])
def test_labels_on_emulation(emu, split, src, fmt, gray):
    G.test_labels_on_every_source_and_canvas(split, gray, src, fmt)


@pytest.mark.parametrize("kind", ["odd", "pixel_seam", "whole"])
def test_synthetic_on_emulation(emu, kind):
    G.test_synthetic_overlays(kind, "nv12", capi.MC_CANVAS_NV12)


def test_yuyv_lanes_and_aligned_on_emulation(emu):
    G.test_labels_on_yuyv_sources(capi.MC_SPLIT_LEFT_RIGHT, False, capi.MC_CANVAS_NV12)
    G.test_lanes_with_hold_and_restart("laplace")
    G.test_aligned_canvases_and_mode_none(capi.MC_CANVAS_BGR)


def test_clear_reset_and_errors_on_emulation(emu):
    G.test_clear_and_reset()
    G.test_errors_keep_the_previous_overlay_and_return_before_any_launch()


def test_labels_with_asynchronous_random_streams():
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "7"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
