"""The Phase stage checkers of tests/test_gpu_phase_stages.py on the CUDA-on-CPU emulation (tests/cuda_emu), at a few
small sizes: the smallest band level the clamp allows, widths of several residues mod 8, an amplify tile just inside
its interior test's right halo, 3 lanes, both staging paths,
the black rectangle (whose NaN runs through amplify, the collapse and the egress), the lane lifecycle and a cutoff
change."""
import pytest

from lvm_b200 import capi
import test_gpu_phase_stages as S

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_stages_on_small_seams(emu):
    S.run_phase(11, 11, 1, n=3)
    S.run_phase(67, 21, 3, n=3, options=(("use_tma", 0),))
    S.run_phase(139, 37, 1, levels=3, n=3, kind="impulses")
    S.run_phase(197, 40, 1, levels=2, n=3)      # amplify: a tile 5 columns short of its 8-pixel right halo


def test_stages_on_the_black_rectangle(emu):
    s = S.run_phase(192, 128, 1, levels=4, n=3, kind="blackrect", oracle=True)
    assert s["nan_patch"] > 0 and s["amp_nan"] > 0 and s["nan_L"] > 0, s
    assert S.run_phase(192, 128, 1, levels=8, n=3, kind="windowbox", oracle=True)["clamp"] > 0


def test_amplify_truncation_and_wavelength_zero(emu):
    assert S.run_phase(70, 39, 1, levels=3, n=3, kind="windowbox", alpha=150, wavelength=80.0)["trunc"] > 0
    S.run_phase(70, 39, 1, levels=3, n=3, kind="windowbox", wavelength=100.0)


def test_lanes_and_cutoff_change(emu):
    events = {2: [("restart", 1), ("hold", 2, 1)], 3: [("hold", 0, 1), ("restart", 1)], 4: [("hold", 0, 0), ("hold", 2, 0)]}
    S.run_phase(65, 32, 3, levels=3, n=6, kind="blackrect", events=events)
    S.run_phase(65, 32, 1, levels=3, n=4, events={2: [("cutoffs", 0.8, 3.0)]})


def test_taps_are_read_only_and_absent_without_a_frame(emu):
    S.test_taps_are_read_only_and_absent_without_a_frame()
