"""mc_set_lane_roi without a GPU: the library exports it, the header declares it, and the ctypes binding matches the
declaration."""
import ctypes as C
import os
import re

from lvm_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "magcore_b200.h")


def test_symbol_is_exported_and_bound_as_declared():
    text = open(HEADER).read()
    assert re.search(r"mc_status\s+mc_set_lane_roi\s*\(\s*mc_handle\s*\*\s*h\s*,\s*int\s+lane\s*,\s*const\s+float\s*\*\s*roi\s*\)\s*;",
                     text)
    restype, args = capi.SIGNATURES["mc_set_lane_roi"]
    assert restype is C.c_int and len(args) == 3
    assert args[1] is C.c_int and args[2]._type_ is C.c_float
    lib = C.CDLL(capi.LIB_PATH)
    assert hasattr(lib, "mc_set_lane_roi")
    assert capi.lib().mc_set_lane_roi(None, 0, None) == capi.MC_ERR_INVALID
