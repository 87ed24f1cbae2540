#!/usr/bin/env python
"""Time of mc_save_lane / mc_load_lane per mode at 1080p colour, into and from pinned (mc_host_alloc) and pageable host
buffers: the median of --repeats blocking calls on a 1-lane handle whose lane holds state, after one warm-up call of each
kind.  Workloads (the blob sizes of include/magcore_b200.h):
  laplace  6 levels (hi / lo of levels 1..5)
  phase    6 levels (13 planes of band levels 0..4) and the lane's filter design
  color    3 levels, a 64-slot window (30 fps), full
Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

    python tools/bench_lane_state.py [--repeats 9]"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card   # noqa: E402

W, H = 1920, 1080


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=9)
    args = ap.parse_args()

    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.synth import synth_frame

    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_state.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    M = L.MagnificationMode
    lib = capi.lib()

    def params(mode, amp, wl, lo, hi, levels):
        return L.toParams(L.MagUiValues(mode=mode, amplification=amp, wavelength=wl, low=lo, high=hi, chroma=0, levels=levels,
                                        captureFps=30.0))

    workloads = {"laplace": (params(M.Laplace, 20, 50.0, 0.4, 3.0, 6), 3),
                 "phase": (params(M.Phase, 50, 50.0, 0.4, 3.0, 6), 3),
                 "color": (params(M.Color, 100, 0.0, 0.8, 1.2, 3), 70)}
    frames = [synth_frame(t, W, H, 3) for t in range(4)]
    results = {}
    for name, (mag, n) in workloads.items():
        m = L.MagnificationProcessor(0, lanes=1)
        cfg = L.ProcessorConfig(magnification=mag)
        for t in range(n):
            m.process_image(frames[t % len(frames)], cfg)
        size = C.c_size_t(0)
        m._check(lib.mc_save_lane(m._h, 0, None, 0, C.byref(size)))
        nbytes = size.value
        pinned_p = lib.mc_host_alloc(nbytes)
        assert pinned_p
        pageable = np.empty(nbytes, np.uint8)
        row = {"blob_MB": nbytes / 1e6}
        for kind, ptr in (("pinned", pinned_p), ("pageable", pageable.ctypes.data)):
            def save():
                m._check(lib.mc_save_lane(m._h, 0, ptr, nbytes, C.byref(size)))

            def load():
                m._check(lib.mc_load_lane(m._h, 0, ptr, nbytes))

            for op, fn in (("save", save), ("load", load)):
                fn()   # warm-up: the handle's staging is allocated here for pageable buffers
                ts = []
                for _ in range(args.repeats):
                    t0 = time.perf_counter()
                    fn()   # blocking: returns after the copies completed
                    ts.append(time.perf_counter() - t0)
                ms = statistics.median(ts) * 1e3
                row[f"{op}_{kind}_ms"] = round(ms, 3)
                row[f"{op}_{kind}_GBps"] = round(nbytes / (ms * 1e-3) / 1e9, 2)
        lib.mc_host_free(pinned_p)
        m.close()
        results[name] = row
        print(name, row)
    after = card()
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')}); after: SM clock {after.get('clocks.sm')}")
    print(json.dumps({"card": before, "card_after": after, "repeats": args.repeats, "results": results}))


if __name__ == "__main__":
    main()
