"""Phase (Riesz) clips (mc_process_clip) on the CUDA-on-CPU emulation (tests/cuda_emu): the analysis, amplification and
synthesis over virtual lanes and the temporal loop of k_riesz_phase_clip, checked bit for bit against frame calls
without a GPU; and the launch count of a clip, which is that of one frame call whatever the clip's length."""
import pytest

from oracle import livim_oracle as O
from lvm_b200 import capi
from test_gpu_clip import check_clip, check_lanes_clip
from test_gpu_lanes import PHASE_UI
from test_gpu_phase_clip import check_launches_per_clip

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_phase_clip_on_emulation(emu):
    """a fresh handle (its passthrough first frame inside the clip), then the continuing one"""
    got = check_clip(O.MODE_PHASE, PHASE_UI, 83, 45, 3, [("clip", 3), ("clip", 3)])
    assert got[0][:, 0].tolist() == [0, 1, 1] and got[1].all()


def test_phase_clip_lanes_on_emulation(emu):
    check_lanes_clip(O.MODE_PHASE, PHASE_UI, 83, 45, 3, lanes=3, restart=2, hold=1, clips=(2, 3, 2))


def test_phase_clip_launch_count_on_emulation(emu):
    check_launches_per_clip()
