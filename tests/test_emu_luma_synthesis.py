"""L-only synthesis of the Laplace path on the CUDA-on-CPU emulation (tests/cuda_emu), at small sizes: the strip egress
and collapses over the L planes only give the tile egress's full synthesis bit for bit, without a GPU."""
import pytest

from lvm_b200 import capi
from test_gpu_luma_synthesis import (check_chroma_switch, check_clips, check_huge_gains, check_lanes, check_shapes,
                                     check_sticky_bound)

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("w,h,lv,band_from_state", [(130, 70, 4, 1), (121, 75, 3, 0), (83, 45, 2, 1)])
def test_luma_synthesis_shapes_on_emulation(emu, w, h, lv, band_from_state):
    check_shapes(w, h, lv, band_from_state, frames=3)


def test_luma_synthesis_lanes_on_emulation(emu):
    check_lanes(83, 45, 3, lanes=4, groups=2)


def test_luma_synthesis_clip_on_emulation(emu):
    check_clips(83, 45, 3, lanes=2, n=3, clips=1)


def test_luma_synthesis_chroma_switch_on_emulation(emu):
    check_chroma_switch(83, 45, 3)


def test_luma_synthesis_sticky_bound_on_emulation(emu):
    check_sticky_bound(83, 45, 3)


def test_luma_synthesis_huge_gains_on_emulation(emu):
    check_huge_gains(83, 45, 3)
