"""Loader for oracle/_ref/_livim_ref — TEST INFRASTRUCTURE ONLY (never imported by the product path).

``_livim_ref`` is the reference's *own* hot-path source (/root/reference/src/processing/**: MagnifyCore.hpp,
SpatialFilter.cpp, TemporalFilter.cpp, RieszPyramid.cpp, ComplexMat.hpp, MagnificationProcessor.cpp,
PreprocessProcessor.cpp, GrayscaleProcessor.cpp, ChainBuilder.cpp, MagnificationParamsUi.hpp) compiled
unmodified, in place, by ``oracle/build_ref.py`` against the cvshim facade, which forwards every pixel operation
to the real OpenCV kernels in cv2.  It pins ``oracle/livim_oracle.py`` (tests/test_ref_pin.py: bit-exact) and is
the CPU arm of ``bench.py`` (``cpu_baseline.kind == "reference"``).

Where the reference sources are absent, a prebuilt module under oracle/_ref/ (git-ignored) is imported as is.
"""
from __future__ import annotations

import importlib.util
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_MOD = None
_TRIED = False


def load(build: bool = True):
    """Returns the _livim_ref module, or None if it is neither built nor buildable here."""
    global _MOD, _TRIED
    if _MOD is not None or _TRIED:
        return _MOD
    _TRIED = True
    try:
        from . import build_ref
    except ImportError:   # imported as a top-level module
        if _HERE not in sys.path:
            sys.path.insert(0, _HERE)
        import build_ref
    path = build_ref.build() if build else (build_ref.module_path() if os.path.exists(build_ref.module_path()) else None)
    if path is None or not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("_livim_ref", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _MOD = mod
    return mod


_MODES = {0: "Laplace", 1: "Phase", 2: "Color", 3: "None_"}


def mode_enum(R, mode: int):
    return getattr(R.MagnificationMode, _MODES[mode])


def to_ref_config(R, ocfg):
    """oracle ProcessorConfig (livim_oracle.py) -> the reference's livim::ProcessorConfig, field by field."""
    cfg = R.ProcessorConfig()
    cfg.grayscale = bool(ocfg.grayscale)
    pp = R.PreprocessParams()
    for k in ("downscale", "roiEnabled", "roiX", "roiY", "roiW", "roiH"):
        setattr(pp, k, getattr(ocfg.preprocess, k))
    cfg.preprocess = pp
    cfg.magnification = to_ref_params(R, ocfg.magnification)
    return cfg


def to_ref_params(R, op):
    mp = R.MagnificationParams()
    mp.mode = mode_enum(R, op.mode)
    for k in ("amplification", "coWavelength", "coLow", "coHigh", "chromAttenuation", "levels", "framerate"):
        setattr(mp, k, getattr(op, k))
    return mp
