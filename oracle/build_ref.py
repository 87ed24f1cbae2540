"""Build oracle/_ref/_livim_ref*.so — TEST INFRASTRUCTURE ONLY.

Compiles the reference's own hot-path sources *where they lie* under /root/reference/src (nothing is copied
into this repo) together with the cvshim facade (oracle/cvshim, forwards to cv2) and the pybind11 bindings
(oracle/ref_binding.cpp).  Outputs go only to oracle/_ref/ (git-ignored).

The reference's real build (CMake + vcpkg OpenCV 4 + Qt 6) cannot run in this image — there are no OpenCV C++
headers or libraries; the only OpenCV present is the statically linked cv2 Python wheel, which exports no C++
symbols — hence the facade.  Compile flags mirror a plain x86-64 release build: -O2, no -march (no FMA
contraction in the reference's own scalar code).
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("LIVIM_REFERENCE_SRC", "/root/reference/src")
OUT_DIR = os.path.join(HERE, "_ref")

# reference translation units on the path (SURVEY.md §8a/§8f-1), relative to REF_SRC
REF_UNITS = [
    "processing/magnification/SpatialFilter.cpp",
    "processing/magnification/TemporalFilter.cpp",
    "processing/magnification/RieszPyramid.cpp",
    "processing/MagnificationProcessor.cpp",
    "processing/PreprocessProcessor.cpp",
    "processing/GrayscaleProcessor.cpp",
    "processing/ChainBuilder.cpp",
]
OWN_UNITS = [os.path.join(HERE, "cvshim", "cvshim.cpp"), os.path.join(HERE, "ref_binding.cpp"), os.path.join(HERE, "mc_dl.cpp")]
ROOT = os.path.dirname(HERE)
ADAPTER_INC = [os.path.join(ROOT, "live-video-magnification_b200", "adapter"), os.path.join(ROOT, "include")]


def module_path() -> str:
    return os.path.join(OUT_DIR, "_livim_ref" + sysconfig.get_config_var("EXT_SUFFIX"))


def reference_present() -> bool:
    return all(os.path.exists(os.path.join(REF_SRC, u)) for u in REF_UNITS)


def build(force: bool = False) -> str | None:
    """Returns the module path, or None when the reference sources are absent and nothing is prebuilt."""
    out = module_path()
    if not reference_present():
        return out if os.path.exists(out) else None
    import pybind11

    srcs = [os.path.join(REF_SRC, u) for u in REF_UNITS] + OWN_UNITS
    deps = srcs + [os.path.join(HERE, "cvshim", "opencv2", h) for h in ("core.hpp", "imgproc.hpp")] + [__file__] + \
        [os.path.join(ADAPTER_INC[0], "MagnificationProcessorB200.hpp"), os.path.join(ADAPTER_INC[1], "magcore_b200.h")]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    obj_dir = os.path.join(OUT_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    flags = ["-O2", "-std=c++20", "-fPIC", "-fvisibility=hidden", "-I", os.path.join(HERE, "cvshim"), "-I", REF_SRC,
             "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], "-I", ADAPTER_INC[0], "-I", ADAPTER_INC[1]]

    def compile_one(src: str) -> str:
        obj = os.path.join(obj_dir, os.path.basename(src).replace(".cpp", ".o"))
        # the facade's own convertTo loops use fmaf (as OpenCV's SIMD convertTo does): give that one unit the FMA
        # instruction so they are not libm calls; the reference's units keep plain x86-64 flags
        own = ["-O3", "-mfma", "-ffp-contract=off"] if src.endswith("cvshim.cpp") else []
        r = subprocess.run(["g++", *flags, *own, "-c", src, "-o", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout)
            raise RuntimeError(f"oracle/_ref: compiling {src} failed")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2)) as ex:
        objs = list(ex.map(compile_one, srcs))
    r = subprocess.run(["g++", "-shared", "-o", out, *objs, "-ldl"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("oracle/_ref: link failed")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
