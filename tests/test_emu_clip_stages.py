"""The clip stage checks of tests/test_gpu_clip_stages.py on the CUDA-on-CPU emulation (tests/cuda_emu), at a few small
sizes: k_level_clip with and without TMA staging over clips that reuse both barrier phases, faithful level 0, state set
to +-1e7 and RUN / FIRST / HOLD lanes in one clip; k_riesz_phase_clip on black content (the NaN patch and the clamp
branch), across a cutoff change at a clip's start with a held lane, and with filter2D's scalar tail columns inside a
tile that starts below them; Color's batched kernels with the extremum in the last virtual lane, a window that wraps
inside a clip, and the output stretch's extremes in the tail columns."""
import pytest

from lvm_b200 import capi
import test_gpu_clip_stages as S

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_laplace_clip_stages(emu):
    S.run_laplace_clips(121, 33, 3, 1, 3, clips=(2, 6), kind="noise", set_state=(1,), co_low=0.0, co_high=1.5)
    S.run_laplace_clips(67, 41, 1, 2, 4, clips=(3, 4), kind="shadows", pad=3, set_state=(1,),
                        options=(("use_tma", 0), ("faithful_level0", 1)))
    events = {1: [("restart", 1), ("hold", 2, 1)], 2: [("hold", 2, 0)]}
    S.run_laplace_clips(69, 35, 3, 3, 4, clips=(2, 3, 2), events=events, chroma=0, set_state=(1,))


def test_phase_clip_stages(emu):
    s = S.run_phase_clips(96, 64, 1, levels=8, clips=(2, 5), kind="windowbox")
    assert s["nan_patch"] > 0 and s["nan_L"] > 0, s
    events = {1: [("cutoffs", 0.8, 3.0), ("restart", 1), ("hold", 2, 1)], 2: [("hold", 2, 0)]}
    S.run_phase_clips(69, 36, 3, levels=4, clips=(2, 3, 3), events=events, options=(("use_tma", 0),))
    # 45 = 40 + 5: the tail columns 40..44 lie in the tile at x0 = 32 (level 1: 23 = 16 + 7, tile x0 = 0)
    S.run_phase_clips(45, 24, 1, levels=4, clips=(1, 3))


def test_color_clip_stages(emu):
    S.flicker_clip(46, 30, 3, 1, 1, 7, 0, 2, 14, 22, 6, 1)
    S.flicker_clip(64, 48, 3, 2, 1, 5, 1, 2, 23, 31, 4, -1)
    kh, *_ = S.run_color_clips(40, 30, 3, 1, (10, 9, 4), fps=(8.0, 8.0, 30.0), lo=0.8, hi=1.2)
    kh.close()
    S.stretch_clip(13, 9, 3, 1, 0, (8, 12, 2), (7, 12, 0))
