"""Host-side mirror of the reference's operator interface for the hot path:
``livim::IProcessor`` / ``livim::MagnificationProcessor`` (reference
src/processing/IProcessor.hpp:10-60, src/processing/MagnificationProcessor.cpp:10-67) and the
parameter structs / UI mapping around it (IProcessor.hpp:14-48, MagnificationParamsUi.hpp:74-103).

Same names, argument meaning and error behaviour as the reference: ``process(frame, cfg)`` returns
the *same* frame object when the reference would return its input FrameRef (identity /
passthrough), otherwise a fresh frame that never aliases the input; a failing core raises (the
caller's firewall then calls ``reset()``, ProcessingChain.cpp:50-62).  All arithmetic happens on
the H100 behind the C ABI (include/magcore_b200.h).
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass, field, replace
from typing import Optional

import numpy as np

from . import capi
from .capi import McParams, MagcoreError

__all__ = ["ProcessingChainB200", "MagnificationMode", "MagnificationParams", "PreprocessParams", "ProcessorConfig", "Frame",
           "IProcessor", "MagnificationProcessor", "toParams", "MagUiValues", "calculateMaxLevels",
           "getOptimalBufferSize", "butterworth", "MagcoreError"]


class MagnificationMode(enum.IntEnum):  # IProcessor.hpp:10
    Laplace = 0
    Phase = 1
    Color = 2
    NONE = 3


@dataclass
class MagnificationParams:  # IProcessor.hpp:14-23
    mode: MagnificationMode = MagnificationMode.Laplace
    amplification: float = 0.0
    coWavelength: float = 0.0
    coLow: float = 0.0
    coHigh: float = 0.0
    chromAttenuation: float = 0.0
    levels: int = 4
    framerate: float = 30.0


@dataclass
class PreprocessParams:  # IProcessor.hpp:26-41
    downscale: int = 1
    roiEnabled: bool = False
    roiX: float = 0.0
    roiY: float = 0.0
    roiW: float = 1.0
    roiH: float = 1.0


@dataclass
class ProcessorConfig:  # IProcessor.hpp:44-48
    grayscale: bool = False
    preprocess: PreprocessParams = field(default_factory=PreprocessParams)
    magnification: MagnificationParams = field(default_factory=MagnificationParams)


@dataclass
class MagUiValues:  # MagnificationParamsUi.hpp:14-23
    mode: MagnificationMode = MagnificationMode.Laplace
    amplification: int = 20
    wavelength: float = 50.0
    low: float = 1.0
    high: float = 2.5
    chroma: int = 0
    levels: int = 4
    captureFps: float = 30.0


@dataclass
class Frame:  # core/Frame.hpp:16-25 (metadata is carried through untouched)
    image: np.ndarray
    seq: int = 0
    ptsUs: int = 0
    captureTs: float = 0.0
    width: int = 0
    height: int = 0
    format: str = "BGR8"


def _to_mc(cfg: ProcessorConfig) -> McParams:
    m, pp = cfg.magnification, cfg.preprocess
    return McParams(int(m.mode), int(m.levels), float(m.amplification), float(m.coWavelength), float(m.coLow),
                    float(m.coHigh), float(m.chromAttenuation), float(m.framerate), int(pp.downscale),
                    int(bool(pp.roiEnabled)), float(pp.roiX), float(pp.roiY), float(pp.roiW), float(pp.roiH))


def toParams(v: MagUiValues) -> MagnificationParams:
    """MagnificationParamsUi.hpp:74-103, evaluated by the core (mc_params_from_ui)."""
    p = McParams()
    capi.lib().mc_params_from_ui(C.byref(p), int(v.mode), int(v.amplification), float(v.wavelength), float(v.low),
                                 float(v.high), int(v.chroma), int(v.levels), float(v.captureFps))
    return MagnificationParams(MagnificationMode(p.mode), p.amplification, p.coWavelength, p.coLow, p.coHigh,
                               p.chromAttenuation, p.levels, p.framerate)


def calculateMaxLevels(width: int, height: int) -> int:
    """SpatialFilter.cpp:5-11."""
    return capi.lib().mc_calculate_max_levels(width, height)


def getOptimalBufferSize(fps: int) -> int:
    """TemporalFilter.cpp:82-94."""
    return capi.lib().mc_optimal_buffer_size(fps)


def butterworth(order: int, wn: float):
    """TemporalFilter.cpp:279-297 -> (a, b)."""
    a = (C.c_double * (order + 1))()
    b = (C.c_double * (order + 1))()
    st = capi.lib().mc_butterworth(order, wn, a, b)
    if st != capi.MC_OK:
        raise MagcoreError(st, "mc_butterworth")
    return list(a), list(b)


class IProcessor:  # IProcessor.hpp:50-60
    def process(self, frame: Frame, cfg: ProcessorConfig) -> Frame:
        raise NotImplementedError

    def reset(self) -> None:
        pass


class MagnificationProcessor(IProcessor):
    """H100 drop-in for livim::MagnificationProcessor.  ``lanes`` > 1 steps that many independent
    streams in lock-step (images then carry a leading lane axis)."""

    def __init__(self, device: int = 0, lanes: int = 1):
        self._lib = capi.lib()
        h = C.c_void_p()
        st = self._lib.mc_create_lanes(device, lanes, C.byref(h))
        if st != capi.MC_OK:
            raise MagcoreError(st, (self._lib.mc_last_error(None) or b"").decode())
        self._h, self.device, self.lanes = h, device, lanes

    # -- lifecycle ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.mc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int):
        if st != capi.MC_OK:
            raise MagcoreError(st, (self._lib.mc_last_error(self._h) or b"").decode())

    def set_option(self, key: str, value: int):
        self._check(self._lib.mc_set_option(self._h, key.encode(), int(value)))

    # -- IProcessor --------------------------------------------------------------------------
    def reset(self) -> None:
        """MagnificationProcessor::reset (MagnificationProcessor.cpp:10-15)."""
        self._check(self._lib.mc_reset(self._h))

    # -- lane lifecycle (multi-stream serving) -----------------------------------------------
    def restart_lane(self, lane: int) -> None:
        """The lane's next frame is its first frame (a stream joins, or hits a scene cut); the other lanes run on.
        On a 1-lane processor this is reset()."""
        self._check(self._lib.mc_restart_lane(self._h, int(lane)))

    def hold_lane(self, lane: int, hold: bool = True) -> None:
        """While held, frame calls skip the lane: its temporal state stays as it is and its output is not written
        (a stream without a new frame this step).  Holds survive reset()."""
        self._check(self._lib.mc_hold_lane(self._h, int(lane), int(bool(hold))))

    def lane_produced(self) -> np.ndarray:
        """-> bool[lanes]: which lanes produced an output in the most recent frame call (or collect())."""
        a = np.zeros(self.lanes, np.uint8)
        self._check(self._lib.mc_lane_produced(self._h, a.ctypes.data_as(C.POINTER(C.c_uint8)), self.lanes))
        return a.astype(bool)

    def process(self, frame: Frame, cfg: ProcessorConfig) -> Frame:
        """MagnificationProcessor::process (MagnificationProcessor.cpp:17-67)."""
        produced, out = self.process_image(frame.image, cfg)
        if not produced:
            return frame  # identity / passthrough: the very same FrameRef
        return replace(frame, image=out, format="BGR8" if out.ndim - (self.lanes > 1) == 3 else "Gray8")

    def _geom(self, image: np.ndarray):
        a = image if self.lanes == 1 else image[0]
        if self.lanes > 1 and image.shape[0] != self.lanes:
            raise ValueError("leading axis must equal lanes")
        h, w = a.shape[:2]
        c = 1 if a.ndim == 2 else a.shape[2]
        return w, h, c

    def process_image(self, image: Optional[np.ndarray], cfg: ProcessorConfig):
        """-> (produced, out8u or the input image).  On a multi-lane processor ``produced`` means "some lane produced",
        and the lanes that did not (held, or passing through) carry their input frame, as the reference returns the
        input FrameRef of that stream."""
        p = _to_mc(cfg)
        produced = C.c_int(0)
        if image is None or image.size == 0:
            self._check(self._lib.mc_process(self._h, None, 0, 0, 3, 0, C.byref(p), None, 0, C.byref(produced)))
            return False, image
        if image.dtype != np.uint8:
            raise TypeError("image must be uint8 (CV_8UC1 / CV_8UC3)")
        w, h, c = self._geom(image)
        img = image if image.flags["C_CONTIGUOUS"] else np.ascontiguousarray(image)
        step = w * c
        out = np.empty_like(img)
        self._check(self._lib.mc_process(self._h, img.ctypes.data, w, h, c, step, C.byref(p), out.ctypes.data, step,
                                         C.byref(produced)))
        if not produced.value:
            return False, image
        if self.lanes > 1:
            idle = ~self.lane_produced()
            if idle.any():
                out[idle] = img[idle]
        return True, out

    def process_clip(self, frames: np.ndarray, cfg: ProcessorConfig):
        """Magnifies T consecutive frames in one call (mc_process_clip): ``frames`` is [T, H, W(, C)], or
        [T, lanes, H, W(, C)] on a multi-lane processor.  -> (produced bool[T, lanes], out of the same shape).  The result
        equals T process_image calls; frames that did not produce carry their input frame."""
        if frames.dtype != np.uint8:
            raise TypeError("frames must be uint8 (CV_8UC1 / CV_8UC3)")
        img = np.ascontiguousarray(frames)
        if self.lanes > 1 and (img.ndim < 4 or img.shape[1] != self.lanes):
            raise ValueError("frames must be [T, lanes, H, W(, C)] on a multi-lane processor")
        if img.ndim < 3:
            raise ValueError("frames must be [T, H, W(, C)]")
        n = img.shape[0]
        per = img.shape[2:] if self.lanes > 1 else img.shape[1:]
        h, w = per[:2]
        c = 1 if len(per) == 2 else per[2]
        p = _to_mc(cfg)
        out = img.copy()
        flags = np.zeros((n, self.lanes), np.uint8)
        self._check(self._lib.mc_process_clip(self._h, img.ctypes.data, n, w, h, c, w * c, C.byref(p), out.ctypes.data,
                                              w * c, flags.ctypes.data_as(C.POINTER(C.c_uint8))))
        return flags.astype(bool), out

    # -- device-resident / pipelined forms (benchmarks, serving) -----------------------------
    def process_clip_device(self, d_in: int, frames: int, w: int, h: int, c: int, in_step: int, cfg_or_params, d_out: int,
                            out_step: int) -> np.ndarray:
        """mc_process_clip_device on raw device pointers -> produced bool[frames, lanes]."""
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        flags = np.zeros((int(frames), self.lanes), np.uint8)
        self._check(self._lib.mc_process_clip_device(self._h, d_in, int(frames), w, h, c, in_step, C.byref(p), d_out, out_step,
                                                     flags.ctypes.data_as(C.POINTER(C.c_uint8))))
        return flags.astype(bool)

    def process_device(self, d_in: int, w: int, h: int, c: int, in_step: int, cfg_or_params, d_out: int,
                       out_step: int) -> bool:
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        produced = C.c_int(0)
        self._check(self._lib.mc_process_device(self._h, d_in, w, h, c, in_step, C.byref(p), d_out, out_step,
                                                C.byref(produced)))
        return bool(produced.value)

    def process_host(self, in_ptr: int, w: int, h: int, c: int, in_step: int, cfg_or_params, out_ptr: int, out_step: int) -> bool:
        """The blocking C call (mc_process) on raw host pointers — what the C++ adapter does per cv::Mat; with page-locked
        buffers (mc_host_alloc, torch pin_memory) the copies go straight to / from HBM."""
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        produced = C.c_int(0)
        self._check(self._lib.mc_process(self._h, in_ptr, w, h, c, in_step, C.byref(p), out_ptr, out_step, C.byref(produced)))
        return bool(produced.value)

    def submit(self, in_ptr: int, w: int, h: int, c: int, in_step: int, cfg_or_params, out_ptr: int, out_step: int):
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        self._check(self._lib.mc_submit(self._h, in_ptr, w, h, c, in_step, C.byref(p), out_ptr, out_step))

    def collect(self) -> bool:
        produced = C.c_int(0)
        self._check(self._lib.mc_collect(self._h, C.byref(produced)))
        return bool(produced.value)

    # -- NV12 frames (video decoder / encoder hand-off); planes are capi.McNv12 -------------------
    def process_nv12_device(self, d_in: capi.McNv12, w: int, h: int, cfg_or_params, d_out: capi.McNv12) -> bool:
        """mc_process_nv12_device on NV12 device planes."""
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        produced = C.c_int(0)
        self._check(self._lib.mc_process_nv12_device(self._h, C.byref(d_in), w, h, C.byref(p), C.byref(d_out), C.byref(produced)))
        return bool(produced.value)

    def process_clip_nv12_device(self, d_in: capi.McNv12, frames: int, w: int, h: int, cfg_or_params,
                                 d_out: capi.McNv12) -> np.ndarray:
        """mc_process_clip_nv12_device -> produced bool[frames, lanes]."""
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        flags = np.zeros((int(frames), self.lanes), np.uint8)
        self._check(self._lib.mc_process_clip_nv12_device(self._h, C.byref(d_in), int(frames), w, h, C.byref(p), C.byref(d_out),
                                                          flags.ctypes.data_as(C.POINTER(C.c_uint8))))
        return flags.astype(bool)

    def submit_nv12(self, in_planes: capi.McNv12, w: int, h: int, cfg_or_params, out_planes: capi.McNv12):
        """mc_submit_nv12 on NV12 host planes (pinned or pageable); collect() returns the frame."""
        p = cfg_or_params if isinstance(cfg_or_params, McParams) else _to_mc(cfg_or_params)
        self._check(self._lib.mc_submit_nv12(self._h, C.byref(in_planes), w, h, C.byref(p), C.byref(out_planes)))

    def sync(self):
        self._check(self._lib.mc_sync(self._h))

    @property
    def stream(self) -> int:
        return self._lib.mc_stream(self._h) or 0

    @property
    def launch_count(self) -> int:
        return int(self._lib.mc_launch_count(self._h))

    def profile_read(self):
        """-> {(kernel, level): (launches, total_ms)} since the last read (option profile_kernels=1)."""
        buf = C.create_string_buffer(1 << 16)
        self._check(self._lib.mc_profile_read(self._h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            k, lvl, n, ms = line.split()
            out[(k, int(lvl))] = (int(n), float(ms))
        return out

    # -- test-only state access --------------------------------------------------------------
    def state_dims(self, name: str, level: int = 0):
        r, c, ch = C.c_int(), C.c_int(), C.c_int()
        self._check(self._lib.mc_state_dims(self._h, name.encode(), level, C.byref(r), C.byref(c), C.byref(ch)))
        return r.value, c.value, ch.value

    def get_state(self, name: str, level: int = 0) -> Optional[np.ndarray]:
        """-> f32 [lanes][channels][rows][cols] or None if the plane does not exist."""
        r, c, ch = self.state_dims(name, level)
        if r == 0:
            return None
        a = np.empty((self.lanes, ch, r, c), np.float32)
        self._check(self._lib.mc_get_state(self._h, name.encode(), level, a.ctypes.data, a.size))
        return a

    def set_state(self, name: str, level: int, value: np.ndarray):
        r, c, ch = self.state_dims(name, level)
        a = np.ascontiguousarray(value, np.float32).reshape(self.lanes, ch, r, c)
        self._check(self._lib.mc_set_state(self._h, name.encode(), level, a.ctypes.data, a.size))

    def float_output(self, w: int, h: int, c: int) -> np.ndarray:
        a = np.empty((self.lanes, h, w, c), np.float32)
        self._check(self._lib.mc_get_float_output(self._h, a.ctypes.data, a.size))
        return a


class ProcessingChainB200:
    """The reference's per-frame chain ``runChainOnce(chain, in, cfg, original)`` (reference
    src/processing/ChainBuilder.cpp:11-29: PreprocessProcessor -> GrayscaleProcessor -> MagnificationProcessor)
    executed on the H100 behind ``mc_chain_process``: the raw frame is uploaded once, ROI crop + INTER_AREA
    downscale and BGR2GRAY run bit-exact on the device, the magnification core runs on their result.

    ``run_chain_once(frame, cfg) -> (cur, original)`` returns the *same* frame object wherever the reference
    returns the same FrameRef (identity stages / passthrough); it needs ``lanes == 1``.  ``process_device`` and
    ``process_nv12_device`` run the chain on device frames of every lane, for one frame or a clip."""

    def __init__(self, device: int = 0, lanes: int = 1):
        self.magnifier = MagnificationProcessor(device=device, lanes=lanes)
        self.lanes = lanes

    def reset(self) -> None:
        """ProcessingChain's recovery path resets every stage (ProcessingChain.cpp:50-62); only the magnifier has state."""
        self.magnifier.reset()

    @staticmethod
    def geometry(cfg: ProcessorConfig, w: int, h: int, c: int) -> "capi.McChainInfo":
        """mc_chain_geometry: what the chain gives a w x h x c frame under cfg, when the magnifier does not produce."""
        p, info = _to_mc(cfg), capi.McChainInfo()
        st = capi.lib().mc_chain_geometry(C.byref(p), int(w), int(h), int(c), int(cfg.grayscale), C.byref(info))
        if st != capi.MC_OK:
            raise MagcoreError(st, "mc_chain_geometry")
        return info

    def process_device(self, d_in: int, frames: int, w: int, h: int, c: int, in_step: int, cfg: ProcessorConfig, d_out: int,
                       out_step: int, d_original: int = 0, original_step: int = 0):
        """mc_chain_process_device on raw device pointers -> (produced bool[frames, lanes], McChainInfo)."""
        m, p, info = self.magnifier, _to_mc(cfg), capi.McChainInfo()
        flags = np.zeros((int(frames), self.lanes), np.uint8)
        m._check(m._lib.mc_chain_process_device(m._h, d_in, int(frames), w, h, c, in_step, C.byref(p), int(cfg.grayscale), d_out,
                                                out_step, d_original or None, original_step,
                                                flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(info)))
        return flags.astype(bool), info

    def process_nv12_device(self, d_in: capi.McNv12, frames: int, w: int, h: int, cfg: ProcessorConfig, d_out: int,
                            out_step: int, d_original: int = 0, original_step: int = 0):
        """mc_chain_process_nv12_device on NV12 device planes -> (produced bool[frames, lanes], McChainInfo)."""
        m, p, info = self.magnifier, _to_mc(cfg), capi.McChainInfo()
        flags = np.zeros((int(frames), self.lanes), np.uint8)
        m._check(m._lib.mc_chain_process_nv12_device(m._h, C.byref(d_in), int(frames), w, h, C.byref(p), int(cfg.grayscale),
                                                     d_out, out_step, d_original or None, original_step,
                                                     flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(info)))
        return flags.astype(bool), info

    def run_chain_once(self, frame: Frame, cfg: ProcessorConfig):
        m = self.magnifier
        p = _to_mc(cfg)
        info = capi.McChainInfo()
        img = frame.image
        if img is None or img.size == 0:
            m._check(m._lib.mc_chain_process(m._h, None, 0, 0, 3, 0, C.byref(p), int(cfg.grayscale), None, 0, None, 0, C.byref(info)))
            return frame, frame
        if img.dtype != np.uint8:
            raise TypeError("image must be uint8")
        img = img if img.flags["C_CONTIGUOUS"] else np.ascontiguousarray(img)
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else img.shape[2]
        out = np.empty(h * w * c, np.uint8)
        orig = np.empty(h * w * c, np.uint8)
        m._check(m._lib.mc_chain_process(m._h, img.ctypes.data, w, h, c, w * c, C.byref(p), int(cfg.grayscale), out.ctypes.data,
                                         out.size, orig.ctypes.data, orig.size, C.byref(info)))

        def view(buf, ww, hh, cc):
            a = buf[:ww * hh * cc]
            return a.reshape(hh, ww).copy() if cc == 1 else a.reshape(hh, ww, cc).copy()

        original = frame if info.orig_is_input else replace(
            frame, image=view(orig, info.orig_w, info.orig_h, info.orig_channels), width=info.orig_w, height=info.orig_h)
        if info.cur_is_input:
            cur = frame
        else:
            cur = replace(frame, image=view(out, info.out_w, info.out_h, info.out_channels), width=info.out_w,
                          height=info.out_h, format="BGR8" if info.out_channels == 3 else "Gray8")
        return cur, original
