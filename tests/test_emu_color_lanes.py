"""Color lanes with their own windows (option "color_lane_lifecycle") on the CUDA-on-CPU emulation (tests/cuda_emu): the
restart, hold and frame-rate cases of tests/test_gpu_color_lanes.py bit for bit against 1-lane handles, and the launch
sets a Color frame records: uniform lanes keep the lock-step composition, lanes whose windows differ in length run one
DFT pair per filtering lane."""
import pytest

from lvm_b200 import capi
from test_gpu_color_lanes import FPS_EVENTS, HOLDS, LIFECYCLE, RESTARTS, check_lanes, color_cfg, fps_steps
from test_gpu_lanes import proc, process_raw, stack

pytestmark = pytest.mark.emu
W, H = 91, 67


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_restart_on_emulation(emu):
    check_lanes(W, H, 3, 3, 34, RESTARTS)


def test_hold_on_emulation(emu):
    check_lanes(W, H, 1, 3, 36, HOLDS)


def test_framerate_change_on_emulation(emu):
    check_lanes(W, H, 3, 3, 34, FPS_EVENTS, fps=fps_steps)


# the kernels of one Color frame at levels 2 on a frame that goes through the bilinear resize
WARM = {("u8_to_planes", 0): 1, ("gauss_down", 0): 1, ("gauss_down", 1): 1, ("ring_append", 0): 1}
FILTER = {("cufft_r2c", 0): 1, ("mask_mul", 0): 1, ("cufft_c2r", 0): 1, ("minmax_window", 0): 1, ("select", 0): 1,
          ("pyrup2x", 0): 1, ("pyrup2x", 1): 1, ("resize", 0): 1, ("minmax_out", 0): 1, ("color_egress", 0): 1}
FULL = {**WARM, **FILTER}


def compositions(lanes, n, events, options):
    p = proc(lanes, (("profile_kernels", 1),) + tuple(options))
    got = []
    for t in range(n):
        for e in events.get(t, []):
            p.hold_lane(e[1], e[2]) if e[0] == "hold" else p.restart_lane(e[1])
        process_raw(p, stack(t, lanes, W, H, 3), color_cfg(8.0))
        got.append({k: v[0] for k, v in p.profile_read().items()})
    p.close()
    return got


def test_uniform_lanes_keep_the_lockstep_launch_set(emu):
    """With or without the option, lanes in lock-step record the composition of a lock-step handle"""
    for options in ((), LIFECYCLE):
        assert compositions(3, 4, {}, options) == [WARM, FULL, FULL, FULL]


def test_staggered_lanes_run_one_dft_pair_per_filtering_lane(emu):
    """Lane 1 restarted at frame 3 (one column: it does not filter), lane 2 held: one lane filters at length 4 — the
    full-batch pair.  Frame 4: lanes 0 and 1 filter at lengths 5 and 2 — one pair each.  A fully held handle launches
    nothing."""
    events = {3: [("restart", 1), ("hold", 2, 1)], 5: [("hold", 0, 1), ("hold", 1, 1)]}
    got = compositions(3, 6, events, LIFECYCLE)
    assert got[3] == FULL
    assert got[4] == {**FULL, ("cufft_r2c", 0): 2, ("cufft_c2r", 0): 2}
    assert got[5] == {}
