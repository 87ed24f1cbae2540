import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a; run with -m gpu)")
    config.addinivalue_line("markers", "emu: kernel-logic check on the CUDA-on-CPU emulation (tests/cuda_emu), no GPU")
    if os.environ.get("MC_EMU") == "1":
        use_emulated_library(asan=os.environ.get("MC_EMU_ASAN") == "1")


def use_emulated_library(asan=False):
    """Points the ctypes binding at tests/cuda_emu/libmagcore_emu.so (the product's kernels compiled for the
    CUDA-on-CPU emulation) so `-m gpu` parity tests can check kernel LOGIC without a GPU:
        MC_EMU=1 python -m pytest tests/test_gpu_laplace.py -m gpu -k small
    Test infrastructure only: the product never does this."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "cuda_emu"))
    import build_emu
    from lvm_b200 import capi
    capi.LIB_PATH = build_emu.build(asan=asan)
    capi._lib = None


@pytest.fixture(scope="session")
def built():
    """The in-tree native libraries (built by __graft_entry__.build(); rebuilt here if missing)."""
    lib = os.path.join(ROOT, "live-video-magnification_b200", "libmagcore_b200.so")
    hc = os.path.join(ROOT, "tests", "hostcheck", "libhostcheck.so")
    if not (os.path.exists(lib) and os.path.exists(hc)):
        import __graft_entry__ as g
        g.build()
    return lib, hc
