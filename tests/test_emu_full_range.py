"""Full-range content on the CUDA-on-CPU emulation (tests/cuda_emu): the exhaustive ingest and egress checks of
tests/test_gpu_full_range.py on the lattice-edge colours E^3, and one full-range parity case per mode.  The emulation's
__dp2a_lo follows the PTX semantics, so this checks the logic of the device branch of the BGR->Lab conversion (and the
"lab16" state's plumbing) without a GPU."""
import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
import test_gpu_full_range as FR

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.parametrize("aligned", [True, False], ids=["72x81", "77x77"])
@pytest.mark.parametrize("name", list(FR.INGEST))
def test_ingest_lab_on_edge_colours_on_emulation(emu, name, aligned):
    FR.check_ingest(name, aligned, edge=True)


@pytest.mark.parametrize("mode", [O.MODE_LAPLACE, O.MODE_PHASE], ids=["laplace", "phase"])
def test_lab16_state_lifecycle_on_emulation(emu, mode):
    FR.check_lab16_lifecycle(mode)


@pytest.mark.parametrize("aligned", [True, False], ids=["72x81", "77x77"])
def test_egress_pixel_stage_on_edge_colours_on_emulation(emu, aligned):
    FR.check_egress_pixel_stage(aligned, edge=True, against_ref=False)


@pytest.mark.parametrize("mname,kind", [("laplace c3 a200 ch100 L4", "blocks"), ("laplace c1 a20 L2", "checker"),
                                        ("phase a150", "corners"), ("color 8fps", "shadows")])
def test_full_range_parity_on_emulation(emu, mname, kind):
    FR.check_parity(mname, kind, 129, 67)
