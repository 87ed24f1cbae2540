"""The device chain on the CUDA-on-CPU emulation (tests/cuda_emu): a 3-lane BGR chain with ROI, fractional downscale and
gray, through frames and clips with a restart and a hold, equals three 1-lane mc_chain_process handles; an NV12 chain equals
the BGR chain on cv2's conversion; and each call launches the magnifier's kernels plus exactly one chain_front."""
import numpy as np
import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
from test_gpu_chain_lanes import MODES, check_chain, device_call, chain_cfg
from test_gpu_lanes import LAPLACE_UI, lane_frame, proc
from test_gpu_nv12 import Dev, Layout

pytestmark = pytest.mark.emu

W, H = 86, 62
FRONT = dict(down=3, roi=(0.1, 0.15, 0.8, 0.75), gray=True)   # 69 x 46 -> 23 x 15: fractional on both axes


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("mname", ["laplace", "phase"])
def test_three_lane_chain_clip_with_restart_and_hold(emu, mname):
    mode, ui = MODES[mname]
    steps = [("cfg", FRONT), ("clip", 2), ("restart", 2), ("hold", 1, 1), ("clip", 2), ("hold", 1, 0), ("frame",)]
    check_chain(mode, ui, W, H, 3, steps, lanes=3, launches=True)


@pytest.mark.parametrize("settings", [FRONT, dict(down=2)], ids=["crop_down_gray", "down"])
def test_nv12_chain_clip_equals_bgr_chain(emu, settings):
    mode, ui = MODES["laplace"]
    steps = [("cfg", settings), ("clip", 2), ("frame",)]
    check_chain(mode, ui, W, H, 3, steps, lanes=2, nv12=Layout(W, H, pitch=W + 3, uv_row=H + 2), launches=True)


def test_launches_are_the_magnifiers_plus_one_front(emu):
    """The chain's launch count over a clip equals a magnifier clip call on the front's output, plus one"""
    lanes, n = 2, 2
    cfg = chain_cfg(O.MODE_LAPLACE, LAPLACE_UI, **FRONT)
    from lvm_b200 import ProcessingChainB200
    ch = ProcessingChainB200(0, lanes=lanes)
    src = np.stack([lane_frame(t, k, W, H, 3) for t in range(n) for k in range(lanes)])
    n0 = ch.magnifier.launch_count
    _, info, out, _ = device_call(ch, cfg, src, n, W, H, 3)
    chain_launches = ch.magnifier.launch_count - n0
    m = proc(lanes)
    d_in = Dev(np.ascontiguousarray(out))
    d_out = Dev(np.zeros_like(out))
    n0 = m.launch_count
    m.process_clip_device(d_in.ptr, n, info.out_w, info.out_h, 1, info.out_w, cfg, d_out.ptr, info.out_w)
    assert chain_launches == m.launch_count - n0 + 1
