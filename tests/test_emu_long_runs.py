"""The long-run checks of tests/test_gpu_long_runs.py on the CUDA-on-CPU emulation (tests/cuda_emu), shorter and at
smaller sizes: Phase past 100 rad of integrated phase within the run's own bound, Laplace through the slow EMA's
transient without drift, Color through every window length with changes after a wrap and on partly filled rings, the same
content as clips on 2 lanes, every pipeline depth, and 64 lanes stepped through pinned submit / collect.  The depth and
64-lane checks run again with asynchronous streams in a random order."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
import test_gpu_long_runs as G

pytestmark = pytest.mark.emu

W, H = 48, 32


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_phase_long_run_on_emulation(emu):
    G.phase_long_run(W, H, 3, 300, 1.3, every=100, min_phase=100.0)
    G.phase_long_run(W, H, 3, 150, 0.7, low=0.02, high=15.0, every=75, min_phase=30.0)


def test_laplace_long_run_on_emulation(emu):
    G.laplace_long_run(W, H, 3, 700, 50, every=25, transient=300, window=150)


def test_color_long_run_on_emulation(emu):
    G.color_long_run(32, 24, 300)      # the first five changes of the schedule, every window length


@pytest.mark.parametrize("mode,n,levels,w,h", [(O.MODE_LAPLACE, 160, 3, 40, 32), (O.MODE_PHASE, 160, 3, 40, 32),
                                                (O.MODE_COLOR, 180, 2, 32, 24)], ids=["laplace", "phase", "color"])
def test_long_clips_on_emulation(emu, mode, n, levels, w, h):
    G.long_clips(mode, w, h, n, levels)


@pytest.mark.parametrize("kind", ["laplace-pageable", "phase-pinned", "laplace-nv12"])
@pytest.mark.parametrize("depth", [1, 2, 5, 16])
def test_depth_on_emulation(emu, kind, depth):
    G.check_depth(kind, depth, 40, 24, n=40)


def test_bench_shape_on_emulation(emu):
    G.bench_shape(64, 48, 64, 6, clip_frames=3, ref_steps=2)


def test_depth_and_lanes_with_asynchronous_random_streams():
    """The depth and 64-lane checks in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": "5"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "depth_on_emulation or bench_shape_on_emulation"], env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
