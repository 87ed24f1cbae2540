"""NV12 calls on the CUDA-on-CPU emulation (tests/cuda_emu): small frames, clips and a 3-lane restart / hold script equal
the BGR path on cv2's conversions bit for bit, and each call launches the BGR call's kernels plus one nv12_to_bgr and
one bgr_to_nv12 (none when nothing produced)."""
import pytest

from lvm_b200 import capi
from test_gpu_nv12 import MODES, Layout, check_nv12

pytestmark = pytest.mark.emu

W, H = 66, 38


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("mname", list(MODES))
def test_frames_and_clips_on_emulation(emu, mname):
    mode, ui = MODES[mname]
    got = check_nv12(mode, ui, W, H, [("clip", 3), ("frame",), ("bgr",), ("frame",), ("clip", 2)], launches=True)
    assert any(g.any() for g in got)


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_three_lanes_restart_and_hold_on_emulation(emu, mname):
    mode, ui = MODES[mname]
    steps = [("frame",), ("restart", 2), ("hold", 1, 1), ("frame",), ("hold", 1, 0), ("restart", 0), ("clip", 2), ("frame",)]
    check_nv12(mode, ui, W, H, steps, lanes=3, layout=Layout(W, H, pitch=W + 3, uv_row=H + 2), launches=True)
