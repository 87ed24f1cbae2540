"""ctypes binding of include/magcore_b200.h (libmagcore_b200.so, built in-tree by
__graft_entry__.build()).  There is no CPU fallback: if the library is missing or no H100 is
visible, constructing a processor raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmagcore_b200.so")

MC_OK, MC_ERR_INVALID, MC_ERR_CUDA, MC_ERR_NO_DEVICE, MC_ERR_UNSUPPORTED, MC_ERR_INTERNAL = 0, 1, 2, 3, 4, 5
MC_MAX_LANES = 4096
MODE_LAPLACE, MODE_PHASE, MODE_COLOR, MODE_NONE = 0, 1, 2, 3


class McParams(C.Structure):
    _fields_ = [
        ("mode", C.c_int32), ("levels", C.c_int32),
        ("amplification", C.c_double), ("coWavelength", C.c_double), ("coLow", C.c_double),
        ("coHigh", C.c_double), ("chromAttenuation", C.c_double), ("framerate", C.c_double),
        ("pre_downscale", C.c_int32), ("pre_roiEnabled", C.c_int32),
        ("pre_roiX", C.c_float), ("pre_roiY", C.c_float), ("pre_roiW", C.c_float), ("pre_roiH", C.c_float),
    ]


class McChainInfo(C.Structure):
    _fields_ = [("cur_is_input", C.c_int32), ("out_w", C.c_int32), ("out_h", C.c_int32), ("out_channels", C.c_int32),
                ("orig_is_input", C.c_int32), ("orig_w", C.c_int32), ("orig_h", C.c_int32), ("orig_channels", C.c_int32),
                ("magnified", C.c_int32)]


class McNv12(C.Structure):
    """mc_nv12: one NV12 frame set (plane pointers are host or device addresses as integers)."""
    _fields_ = [("y", C.c_void_p), ("uv", C.c_void_p), ("pitch", C.c_size_t), ("lane_stride", C.c_size_t)]


# name -> (restype, argtypes); every symbol include/magcore_b200.h declares
_u8p, _f32p, _vp = C.POINTER(C.c_uint8), C.POINTER(C.c_float), C.c_void_p
_PP = C.POINTER(McParams)
_NV = C.POINTER(McNv12)
SIGNATURES = {
    "mc_abi_version": (C.c_int, []),
    "mc_device_count": (C.c_int, []),
    "mc_params_default": (None, [_PP]),
    "mc_params_from_ui": (None, [_PP, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, C.c_double]),
    "mc_calculate_max_levels": (C.c_int, [C.c_int, C.c_int]),
    "mc_optimal_buffer_size": (C.c_int, [C.c_int]),
    "mc_butterworth": (C.c_int, [C.c_uint, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "mc_motion_gains": (C.c_int, [_PP, C.c_int, C.c_int, C.c_int, _f32p]),
    "mc_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "mc_create_lanes": (C.c_int, [C.c_int, C.c_int, C.POINTER(_vp)]),
    "mc_destroy": (None, [_vp]),
    "mc_reset": (C.c_int, [_vp]),
    "mc_restart_lane": (C.c_int, [_vp, C.c_int]),
    "mc_hold_lane": (C.c_int, [_vp, C.c_int, C.c_int]),
    "mc_lane_produced": (C.c_int, [_vp, _u8p, C.c_int]),
    "mc_process": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, _vp, C.c_size_t, C.POINTER(C.c_int)]),
    "mc_process_device": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, _vp, C.c_size_t, C.POINTER(C.c_int)]),
    "mc_sync": (C.c_int, [_vp]),
    "mc_process_clip_device": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, _vp, C.c_size_t, _u8p]),
    "mc_process_clip": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, _vp, C.c_size_t, _u8p]),
    "mc_chain_process": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, C.c_int, _vp, C.c_size_t, _vp,
                                   C.c_size_t, C.POINTER(McChainInfo)]),
    "mc_chain_geometry": (C.c_int, [_PP, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(McChainInfo)]),
    "mc_chain_process_device": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, C.c_int, _vp, C.c_size_t,
                                          _vp, C.c_size_t, _u8p, C.POINTER(McChainInfo)]),
    "mc_chain_process_nv12_device": (C.c_int, [_vp, _NV, C.c_int, C.c_int, C.c_int, _PP, C.c_int, _vp, C.c_size_t, _vp,
                                               C.c_size_t, _u8p, C.POINTER(McChainInfo)]),
    "mc_pipeline_depth": (C.c_int, [_vp]),
    "mc_submit": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_size_t, _PP, _vp, C.c_size_t]),
    "mc_collect": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "mc_process_nv12_device": (C.c_int, [_vp, _NV, C.c_int, C.c_int, _PP, _NV, C.POINTER(C.c_int)]),
    "mc_process_clip_nv12_device": (C.c_int, [_vp, _NV, C.c_int, C.c_int, C.c_int, _PP, _NV, _u8p]),
    "mc_submit_nv12": (C.c_int, [_vp, _NV, C.c_int, C.c_int, _PP, _NV]),
    "mc_host_alloc": (_vp, [C.c_size_t]),
    "mc_host_free": (None, [_vp]),
    "mc_stream": (_vp, [_vp]),
    "mc_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int]),
    "mc_state_dims": (C.c_int, [_vp, C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mc_get_state": (C.c_int, [_vp, C.c_char_p, C.c_int, _vp, C.c_size_t]),
    "mc_set_state": (C.c_int, [_vp, C.c_char_p, C.c_int, _vp, C.c_size_t]),
    "mc_get_float_output": (C.c_int, [_vp, _vp, C.c_size_t]),
    "mc_launch_count": (C.c_uint64, [_vp]),
    "mc_profile_read": (C.c_int, [_vp, C.c_char_p, C.c_size_t]),
    "mc_last_error": (C.c_char_p, [_vp]),
}

_lib = None


def lib() -> C.CDLL:
    """Loads the in-tree shared library (fails loudly if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback for the magnification core.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype, fn.argtypes = res, args
        _lib = l
    return _lib


class MagcoreError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"magcore status {status}: {msg}")
        self.status = status
