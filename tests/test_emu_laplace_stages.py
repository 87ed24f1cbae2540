"""The Laplace stage checkers of tests/test_gpu_laplace_stages.py on the CUDA-on-CPU emulation (tests/cuda_emu), at a few
small sizes: a width one past the 120-column strip seam, an exact 64 x 32 tile, sizes odd at every level, gray and colour,
3 lanes in two lane groups, both staging paths, both band sources, the tile egress, faithful level 0, L-only synthesis,
the EMA from state set with mc_set_state, and the lane lifecycle."""
import pytest

from lvm_b200 import capi
import test_gpu_laplace_stages as S

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_stages_on_small_seams(emu):
    assert S.run_laplace(121, 33, 3, 1, 3, n=3, kind="noise", sensitivity=True)["sens0"] >= 2 ** 10
    S.run_laplace(128, 64, 1, 3, 4, n=3, kind="noise", options=(("band_from_state", 0), ("lane_groups", 2)))
    S.run_laplace(129, 65, 3, 1, 8, n=3, kind="checker", chroma=0, options=(("use_tma", 0),))
    S.run_laplace(67, 41, 3, 1, 4, n=3, kind="blocks", options=(("faithful_level0", 1), ("egress_strip", 0)), pad=3)


def test_ema_from_set_state(emu):
    S.run_laplace(70, 37, 3, 1, 4, n=3, set_state_at=1, co_low=0.0, co_high=1.5)
    S.run_laplace(70, 37, 1, 1, 3, n=3, set_state_at=1, co_low=0.2, co_high=0.9, options=(("band_from_state", 0),))


def test_lanes_run_first_and_hold(emu):
    events = {2: [("restart", 1), ("hold", 2, 1)], 3: [("hold", 2, 0)]}
    S.run_laplace(69, 35, 3, 3, 4, n=4, events=events, options=(("band_from_state", 0),))


def test_taps_are_read_only_and_absent_without_a_frame(emu):
    S.test_taps_are_read_only_and_absent_without_a_frame()
