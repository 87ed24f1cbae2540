#!/usr/bin/env python
"""Frames/s of a multi-lane handle whose lanes all share the call's parameters ("uniform") against the same handle with a
different mc_set_lane_params override on every lane ("per_lane"), alternated in windows of at least `--window` seconds,
median of `--repeats`.  Device-resident frames, mc_process_device plus a synchronise per step.  Workloads:
  laplace     64 lanes of 1080p Laplace at 6 levels (bench.py's shape and parameters); per_lane mixes chroma 0 and 50
  laplace_l   the same with every lane at chroma 0, so that L-only synthesis stays on and the row isolates the table
  phase       16 lanes of 1080p Phase, per-lane cutoffs, amplifications and frame rates
  color       16 lanes of 1080p Color at 3 levels (option color_lane_lifecycle), per_lane at 25 / 30 / 60 fps (windows
              64 / 64 / 128)
Prints the card's name, power limit and SM clocks
read in the same run, and one JSON line.

    python tools/bench_lane_params.py [--window 1.0] [--repeats 3]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card, timed   # noqa: E402

W, H = 1920, 1080


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.synth import synth_frame

    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_params.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    M = L.MagnificationMode

    def params(mode, amp, wl, lo, hi, chroma, levels, fps):
        return L.toParams(L.MagUiValues(mode=mode, amplification=amp, wavelength=wl, low=lo, high=hi, chroma=chroma,
                                        levels=levels, captureFps=fps))

    workloads = {
        "laplace": (M.Laplace, 64, params(M.Laplace, 20, 50.0, 0.4, 3.0, 0, 6, 30.0),
                    lambda k: params(M.Laplace, 5 + k % 30, 20.0 + k, 0.2 + 0.01 * k, 2.0 + 0.05 * k, [0, 50][k % 2], 6,
                                     [25.0, 30.0, 60.0][k % 3])),
        "laplace_l": (M.Laplace, 64, params(M.Laplace, 20, 50.0, 0.4, 3.0, 0, 6, 30.0),
                      lambda k: params(M.Laplace, 5 + k % 30, 20.0 + k, 0.2 + 0.01 * k, 2.0 + 0.05 * k, 0, 6,
                                       [25.0, 30.0, 60.0][k % 3])),
        "phase": (M.Phase, 16, params(M.Phase, 50, 50.0, 0.4, 3.0, 0, 4, 30.0),
                  lambda k: params(M.Phase, 30 + 3 * k, 40.0 + k, 0.3 + 0.02 * k, 2.0 + 0.1 * k, 0, 4, [25.0, 30.0, 60.0][k % 3])),
        "color": (M.Color, 16, params(M.Color, 100, 0.0, 0.8, 1.2, 0, 3, 30.0),
                  lambda k: params(M.Color, 100, 0.0, 0.8, 1.2, 0, 3, [25.0, 30.0, 60.0][k % 3])),
    }
    results = {}
    for name, (mode, lanes, base, lane_params) in workloads.items():
        frames = torch.from_numpy(np.stack([synth_frame(k % 8, W, H, 3, seed=k) for k in range(lanes)])).cuda()
        out = torch.empty_like(frames)
        cfg = L.ProcessorConfig(magnification=base)
        handles = {"uniform": L.MagnificationProcessor(0, lanes=lanes), "per_lane": L.MagnificationProcessor(0, lanes=lanes)}
        for p in handles.values():
            p.set_option("color_lane_lifecycle", 1)
        for k in range(lanes):
            handles["per_lane"].set_lane_params(k, lane_params(k))

        def step(p):
            p.process_device(frames.data_ptr(), W, H, 3, W * 3, cfg, out.data_ptr(), W * 3)
            torch.cuda.synchronize()

        for p in handles.values():   # warm-up: allocation, the Color window's fill
            for _ in range(140):
                step(p)
        rates = {k: [] for k in handles}
        for _ in range(args.repeats):
            for key, p in handles.items():
                n, dt = timed(lambda i: step(p), args.window)
                rates[key].append(n * lanes / dt)
        results[name] = {k: round(statistics.median(v), 1) for k, v in rates.items()}
        for p in handles.values():
            p.close()
        print(f"{name:9s} lanes={lanes:2d}  " + "  ".join(f"{k}={v}" for k, v in results[name].items()), flush=True)
    print(json.dumps({"card": before, "card_after": card(), "frames_per_s": results}))


if __name__ == "__main__":
    main()
