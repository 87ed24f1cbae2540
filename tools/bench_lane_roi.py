#!/usr/bin/env python
"""Frames/s of multi-camera serving where every camera has its own region of interest: 64 lanes of 4K (3840 x 2160)
device frames, each cropped to its own 1920 x 1080 window, Laplace at 6 levels, one chain call plus a synchronise per
step.  Three ways to run it, alternated in windows of at least `--window` seconds, median of `--repeats`:
  per_lane   one 64-lane handle, each lane with its own ROI (mc_set_lane_roi): the front reads per-lane origins
  shared     the same 64-lane handle shape with one ROI for every lane: the cost of the per-lane origins is the gap
  handles    64 one-lane handles, each with its camera's ROI in its call: what serving from one handle gains
Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

    python tools/bench_lane_roi.py [--window 1.0] [--repeats 3]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card, timed   # noqa: E402

W, H, CW, CH, LANES = 3840, 2160, 1920, 1080, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200.synth import synth_frame

    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_roi.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    M = L.MagnificationMode
    mag = L.toParams(L.MagUiValues(mode=M.Laplace, amplification=20, wavelength=50.0, low=0.4, high=3.0, chroma=0, levels=6,
                                   captureFps=30.0))
    # lane k's window: an 8 x 8 grid of origins over the frame's top-left quarter, so every crop is 1920 x 1080
    rois = [((k % 8) * 240 / W, (k // 8) * 135 / H, CW / W, CH / H) for k in range(LANES)]

    def cfg_of(roi):
        return L.ProcessorConfig(magnification=mag, preprocess=L.PreprocessParams(1, True, *roi))

    base = [torch.from_numpy(synth_frame(t, W, H, 3)).cuda() for t in range(8)]   # 8 distinct 4K frames, built once
    frames = torch.stack([base[k % 8] for k in range(LANES)])
    out = torch.empty((LANES, CH, CW * 3), dtype=torch.uint8, device="cuda")
    lane_bytes, out_bytes = W * H * 3, CW * CH * 3
    shared_cfg = cfg_of(rois[0])

    per_lane, shared = L.ProcessingChainB200(0, lanes=LANES), L.ProcessingChainB200(0, lanes=LANES)
    for k, r in enumerate(rois):
        per_lane.set_lane_roi(k, r)
    singles = [L.ProcessingChainB200(0, lanes=1) for _ in range(LANES)]
    single_cfgs = [cfg_of(r) for r in rois]

    def many(ch):
        return lambda i: (ch.process_device(frames.data_ptr(), 1, W, H, 3, W * 3, shared_cfg, out.data_ptr(), CW * 3),
                          torch.cuda.synchronize())

    def one_per_camera(i):
        for k, ch in enumerate(singles):
            ch.process_device(frames.data_ptr() + k * lane_bytes, 1, W, H, 3, W * 3, single_cfgs[k], out.data_ptr() + k * out_bytes,
                              CW * 3)
        torch.cuda.synchronize()

    runs = {"per_lane": many(per_lane), "shared": many(shared), "handles": one_per_camera}
    for f in runs.values():   # warm-up: allocation, module load
        for i in range(10):
            f(i)
    rates = {k: [] for k in runs}
    for _ in range(args.repeats):
        for key, f in runs.items():
            n, dt = timed(f, args.window)
            rates[key].append(n * LANES / dt)
    results = {k: round(statistics.median(v), 1) for k, v in rates.items()}
    print("  ".join(f"{k}={v}" for k, v in results.items()), flush=True)
    print(json.dumps({"card": before, "card_after": card(), "lanes": LANES, "source": [W, H], "crop": [CW, CH],
                      "frames_per_s": results}))


if __name__ == "__main__":
    main()
