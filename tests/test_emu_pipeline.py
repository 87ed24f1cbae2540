"""The pipelined host path (mc_submit / mc_submit_nv12 / mc_collect) on the CUDA-on-CPU emulation (tests/cuda_emu): BGR
and NV12 frame sets, pinned and pageable, with restarts and holds taken at submit, equal the blocking and device calls
bit for bit.  The same checks run again with asynchronous streams in a random order, where an upload, download or
staging buffer that is not ordered by a stream or an event wait gives wrong bytes."""
import os
import subprocess
import sys

import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
from test_gpu_lanes import LAPLACE_UI, PHASE_UI, check_pipelined
from test_gpu_nv12 import check_submit_nv12

pytestmark = pytest.mark.emu

W, H = 66, 38


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("mname", ["laplace", "phase"])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("layout", ["packed", "uv_offset"])
def test_submit_nv12_on_emulation(emu, mname, pinned, layout):
    check_submit_nv12(mname, pinned, layout, W, H)


@pytest.mark.parametrize("mode,ui,pinned", [(O.MODE_LAPLACE, LAPLACE_UI, False), (O.MODE_LAPLACE, LAPLACE_UI, True),
                                            (O.MODE_PHASE, PHASE_UI, False), (O.MODE_PHASE, PHASE_UI, True)])
def test_submit_bgr_on_emulation(emu, mode, ui, pinned):
    check_pipelined(mode, ui, pinned, W, H)


@pytest.mark.parametrize("seed", ["3", "11"])
def test_submit_with_asynchronous_random_streams(seed):
    """The tests above in a fresh process: the emulation reads CUDA_EMU_ASYNC once per process."""
    env = {**os.environ, "CUDA_EMU_ASYNC": "1", "CUDA_EMU_ORDER": "random", "CUDA_EMU_SEED": seed}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "on_emulation"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
