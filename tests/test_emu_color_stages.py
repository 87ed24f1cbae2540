"""The Color stage checkers of tests/test_gpu_color_stages.py on the CUDA-on-CPU emulation (tests/cuda_emu), at a handful
of small sizes: a smallest level of 3 x 3, a width of 3 mod 4, a 3-lane handle with odd (padded) lane blocks, one
extremum-in-the-tail case per reduction and the byte-exact output stretch at amplification 0."""
import pytest

from lvm_b200 import capi
import test_gpu_color_stages as S

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_stages_down_to_a_3x3_level(emu):
    S.run_stages(11, 9, 3, 1, pad=3, oracle=True)
    S.run_stages(33, 41, 1, 2, n=4, oracle=True)


def test_stages_with_padded_lanes_and_resize(emu):
    """91 x 67, levels 2: 3 x 23 x 17 signals a lane (odd), the pyrUp chain ends at 92 x 68"""
    assert S.run_stages(91, 67, 3, 3, levels=2, n=4, oracle=True) == [4, 15, 15, 15]


def test_taps_are_read_only_and_absent_without_a_frame(emu):
    S.test_taps_are_read_only_and_absent_without_a_frame()


def test_window_restart_hold_and_framerate_change(emu):
    S.test_window_per_lane_restart_and_hold()
    S.drive_window(40, 30, 1, 2, [8.0] * 18 + [30.0] * 3 + [8.0] * 3)


def test_mask_edges_on_packed_indices_and_an_empty_band(emu):
    S.test_filter_mask_cases(8.0, 1.0, 2.0)
    S.test_filter_mask_cases(8.0, 1.2, 0.8)


def test_window_extremum_in_the_tail(emu):
    S.flicker_case(24, 16, 3, 1, 1, 7, 0, 2, 7, 11, 6, 1)        # vector path, last element
    S.flicker_case(46, 30, 1, 3, 1, 7, 2, 0, 14, 22, 6, -1)      # scalar path, padded lanes, last lane
    S.test_extremum_in_the_last_vector_of_a_chunk(2)


def test_output_stretch_is_byte_exact_with_the_extremes_in_the_tail(emu):
    S.test_stretch_with_the_extremes_in_the_tail_columns_and_last_row(15, 3)
    S.test_stretch_last_lane_of_3()
