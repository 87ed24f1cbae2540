"""Build and load oracle/_ref/_exporter_ref*.so — TEST INFRASTRUCTURE ONLY.

The reference exporter's own canvas, compose(orig, proc, split, overlay) of export/Exporter.cpp with its drawLabel labels,
compiled in place from /root/reference/src (nothing is copied into this repo) against the facade in this directory,
which forwards every pixel operation to the real OpenCV kernels in cv2.  Output goes only to oracle/_ref/ (git-ignored).
It pins lvm_b200.labels (tests/test_labels_host.py).  Where the reference sources are absent, a prebuilt module under
oracle/_ref/ is loaded as is.
"""
from __future__ import annotations

import importlib.util
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("LIVIM_REFERENCE_SRC", "/root/reference/src")
OUT_DIR = os.path.join(os.path.dirname(HERE), "_ref")
REF_UNIT = "export/Exporter.cpp"   # included by binding.cpp: compose() sits in an anonymous namespace
OWN_UNITS = [os.path.join(HERE, "binding.cpp"), os.path.join(HERE, "facade.cpp")]
HEADERS = [os.path.join(HERE, "opencv2", h) for h in ("core.hpp", "imgproc.hpp", "videoio.hpp")]
_MOD, _TRIED = None, False


def module_path() -> str:
    return os.path.join(OUT_DIR, "_exporter_ref" + sysconfig.get_config_var("EXT_SUFFIX"))


def build(force: bool = False) -> str | None:
    """Returns the module path, or None when the reference sources are absent and nothing is prebuilt."""
    out = module_path()
    if not os.path.exists(os.path.join(REF_SRC, REF_UNIT)):
        return out if os.path.exists(out) else None
    deps = [os.path.join(REF_SRC, REF_UNIT), *OWN_UNITS, *HEADERS, __file__]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    import pybind11

    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = ["g++", "-O2", "-std=c++20", "-fPIC", "-shared", "-fvisibility=hidden", "-I", HERE, "-I", REF_SRC,
           "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], *OWN_UNITS, "-o", out]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("oracle/_ref/_exporter_ref did not build")
    return out


def load(build_it: bool = True):
    """Returns the _exporter_ref module, or None if it is neither built nor buildable here."""
    global _MOD, _TRIED
    if _MOD is not None or _TRIED:
        return _MOD
    _TRIED = True
    path = build() if build_it else (module_path() if os.path.exists(module_path()) else None)
    if path is None or not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("_exporter_ref", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _MOD = mod
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
