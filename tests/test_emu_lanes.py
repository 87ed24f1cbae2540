"""Lane lifecycle (restart / hold of one lane of a multi-lane handle) on the CUDA-on-CPU emulation (tests/cuda_emu):
the per-lane op handling of the Laplace and Phase kernels, checked bit for bit against 1-lane handles without a GPU."""
import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
from test_gpu_lanes import LAPLACE_UI, PHASE_UI, check_hold, check_restart

pytestmark = pytest.mark.emu


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def test_laplace_restart_and_hold_on_emulation(emu):
    check_restart(O.MODE_LAPLACE, LAPLACE_UI, 83, 45, 3, lanes=3, lane=1, at=2, n=4)
    check_hold(O.MODE_LAPLACE, LAPLACE_UI, 83, 45, 3, lanes=3, lane=1, span=(1, 3), n=5)


def test_phase_restart_and_hold_on_emulation(emu):
    check_restart(O.MODE_PHASE, PHASE_UI, 80, 60, 3, lanes=3, lane=1, at=2, n=4)
    check_hold(O.MODE_PHASE, PHASE_UI, 80, 60, 3, lanes=3, lane=1, span=(1, 3), n=5)
