"""Clips of the Laplace path (mc_process_clip) on the CUDA-on-CPU emulation (tests/cuda_emu): the batched ingest and
synthesis over virtual lanes and the temporal loop of k_level_clip, checked bit for bit against frame calls without a GPU."""
import pytest

from oracle import livim_oracle as O
from lvm_b200 import capi
from test_gpu_clip import check_clip, check_lanes_clip, laplace_ui

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_on_emulation(emu, c):
    check_clip(O.MODE_LAPLACE, laplace_ui(3), 83, 45, c, [("clip", 3), ("clip", 3)])


@pytest.mark.parametrize("c", [3, 1])
def test_laplace_clip_lanes_on_emulation(emu, c):
    check_lanes_clip(O.MODE_LAPLACE, laplace_ui(3), 83, 45, c, lanes=3, restart=2, hold=1, clips=(2, 3, 2))
