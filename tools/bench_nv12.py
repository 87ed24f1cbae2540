#!/usr/bin/env python
"""NV12 against BGR frames on the bench workload (1080p Laplace, 6 levels, 64 lanes): one process alternates, in
windows of at least `--window` seconds, median of `--repeats`:
  e2e    mc_submit (pinned BGR, 6.2 MB per frame each way) against mc_submit_nv12 (pinned NV12, 3.1 MB), depth 3;
  device mc_process_device against mc_process_nv12_device on frames resident in HBM;
  the two conversion kernels' device time per frame (profile_kernels, a separate pass);
  a kernel-free copy ceiling: pinned host <-> device on two concurrent streams, at NV12 and at BGR byte counts.
Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

    python tools/bench_nv12.py [--lanes 64] [--window 1.0] [--repeats 3]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"error": "nvidia-smi unavailable"}


def timed(fn, window):
    """Calls fn(k) for k = 0, 1, ... until `window` seconds have passed (fn ends in a synchronise) -> (calls, seconds)."""
    t0, n = time.perf_counter(), 0
    while True:
        fn(n)
        n += 1
        dt = time.perf_counter() - t0
        if dt >= window:
            return n, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=64)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from bench import H, UI, W, make_clip

    if not torch.cuda.is_available():
        raise SystemExit("bench_nv12.py needs an H100: the magnification core has no CPU fallback")
    lanes, T, depth = args.lanes, 2, 3
    before = card()
    p = capi.McParams()
    capi.lib().mc_params_from_ui(C.byref(p), capi.MODE_LAPLACE, UI["amplification"], UI["wavelength"], UI["low"], UI["high"],
                                 UI["chroma"], UI["levels"], UI["fps"])
    bgr = make_clip(T, lanes)

    def nv12(f):
        i420, n = cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420).ravel(), W * H
        uv = np.stack([i420[n:n + n // 4], i420[n + n // 4:]], -1).reshape(H // 2, W)
        return np.concatenate([i420[:n].reshape(H, W), uv])

    nv = np.stack([np.stack([nv12(f) for f in lanes_]) for lanes_ in bgr])   # [T][lanes][3H/2][W]
    row, lane_nv = W * 3, W * H * 3 // 2
    planes = lambda base: capi.McNv12(base, base + W * H, W, lane_nv)

    proc = L.MagnificationProcessor(0, lanes=lanes)
    bgr_p, nv_p = torch.from_numpy(bgr).pin_memory(), torch.from_numpy(nv).pin_memory()
    bgr_out = [torch.empty(bgr.shape[1:], dtype=torch.uint8).pin_memory() for _ in range(depth)]
    nv_out = [torch.empty(nv.shape[1:], dtype=torch.uint8).pin_memory() for _ in range(depth)]
    bgr_d, nv_d = torch.from_numpy(bgr).cuda(), torch.from_numpy(nv).cuda()
    bgr_dout = torch.empty(bgr.shape[1:], dtype=torch.uint8, device="cuda")
    nv_dout = torch.empty(nv.shape[1:], dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    steps = 30   # calls per timed chunk: keeps the pipeline full between the synchronising ends of a chunk

    def e2e(submit):
        def run(k):
            done = 0
            for i in range(steps):
                if i - done >= depth:
                    assert proc.collect(); done += 1
                submit(k * steps + i)
            while done < steps:
                assert proc.collect(); done += 1
        return run

    e2e_bgr = e2e(lambda i: proc.submit(bgr_p[i % T].data_ptr(), W, H, 3, row, p, bgr_out[i % depth].data_ptr(), row))
    e2e_nv = e2e(lambda i: proc.submit_nv12(planes(nv_p[i % T].data_ptr()), W, H, p, planes(nv_out[i % depth].data_ptr())))

    def dev(call):
        def run(k):
            for i in range(steps):
                assert call(k * steps + i)
            proc.sync()
        return run

    dev_bgr = dev(lambda i: proc.process_device(bgr_d[i % T].data_ptr(), W, H, 3, row, p, bgr_dout.data_ptr(), row))
    dev_nv = dev(lambda i: proc.process_nv12_device(planes(nv_d[i % T].data_ptr()), W, H, p, planes(nv_dout.data_ptr())))

    def copies(nbytes):
        h_in = [torch.empty(nbytes, dtype=torch.uint8).pin_memory().fill_(1) for _ in range(depth)]
        h_out = [torch.empty(nbytes, dtype=torch.uint8).pin_memory() for _ in range(depth)]
        d = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(2 * depth)]
        s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()

        def run(k):
            for i in range(steps):
                with torch.cuda.stream(s_in):
                    d[i % depth].copy_(h_in[i % depth], non_blocking=True)
                with torch.cuda.stream(s_out):
                    h_out[i % depth].copy_(d[depth + i % depth], non_blocking=True)
            torch.cuda.synchronize()
        return run

    paths = {"e2e_bgr": e2e_bgr, "e2e_nv12": e2e_nv, "device_bgr": dev_bgr, "device_nv12": dev_nv,
             "copy_ceiling_nv12": copies(lanes * lane_nv), "copy_ceiling_bgr": copies(lanes * H * row)}
    for fn in paths.values():   # warm-up: module load, slot and staging allocation, the first frames' state
        fn(0)
    rates = {k: [] for k in paths}
    for _ in range(args.repeats):
        for k, fn in paths.items():
            n, dt = timed(fn, args.window)
            rates[k].append(n * steps * lanes / dt)
    fps = {k: statistics.median(v) for k, v in rates.items()}

    # the conversion kernels' device time: a pass of its own with per-launch events
    proc.set_option("profile_kernels", 1)
    proc.profile_read()
    n_prof = 20
    for i in range(n_prof):
        proc.process_nv12_device(planes(nv_d[i % T].data_ptr()), W, H, p, planes(nv_dout.data_ptr()))
    prof = proc.profile_read()
    proc.set_option("profile_kernels", 0)
    kern_us = {k: 1e3 * prof[(k, 0)][1] / (prof[(k, 0)][0] * lanes) for k in ("nv12_to_bgr", "bgr_to_nv12")}
    floor_us = 4.5 * W * H / 3.35e12 * 1e6   # 4.5 B/px at the data-sheet 3.35 TB/s
    after = card()
    proc.close()

    result = {
        "workload": f"Laplace {W}x{H}, {UI['levels']} levels, {lanes} lanes, pinned host frames, depth {depth}",
        "frames_per_s": {k: round(v, 1) for k, v in fps.items()},
        "e2e_nv12_over_bgr": round(fps["e2e_nv12"] / fps["e2e_bgr"], 3),
        "copy_ceiling_nv12_over_bgr": round(fps["copy_ceiling_nv12"] / fps["copy_ceiling_bgr"], 3),
        "e2e_nv12_share_of_nv12_ceiling": round(fps["e2e_nv12"] / fps["copy_ceiling_nv12"], 3),
        "kernel_us_per_frame": {k: round(v, 3) for k, v in kern_us.items()},
        "kernel_bytes_per_frame": 4.5 * W * H,
        "kernel_floor_us_at_3.35TBps": round(floor_us, 3),
        "window_s": args.window, "repeats": args.repeats,
        "card_before": before, "card_after": after,
    }
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')})", flush=True)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
