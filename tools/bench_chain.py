#!/usr/bin/env python
"""The processing chain's front on a 4K source (the README's advice for a machine that cannot keep up: downscale): 3840 x
2160 frames, downscale 2, 1080p Laplace at 6 levels, 16 lanes, in frame calls and in clips of 16.  One process alternates,
in windows of at least `--window` seconds, median of `--repeats`, three ways to get there:
  nv12_fused    mc_chain_process_nv12_device: NV12 in, the front converts inside its tap walk;
  nv12_convert  mc_debug_nv12_to_bgr at 4K first (the conversion kernel, synchronised), then mc_chain_process_device;
  bgr           mc_chain_process_device on 4K BGR frames.
Every call writes the original tap (d_original), as an exporter composing `cur` with `original` does.  A separate pass with
profile_kernels reads the chain_front kernel's device time per frame (and the 4K conversion's, timed with CUDA events), set
against the bytes the kernel has to move at the data-sheet 3.35 TB/s.  Prints the card's name, power limit and SM clocks
read in the same run, and one JSON line.

    python tools/bench_chain.py [--lanes 16] [--clip 16] [--window 1.0] [--repeats 3]"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card, timed   # noqa: E402

SW, SH, DOWN, LEVELS = 3840, 2160, 2, 6
DW, DH = SW // DOWN, SH // DOWN
PEAK = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=16)
    ap.add_argument("--clip", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.synth import synth_frame

    if not torch.cuda.is_available():
        raise SystemExit("bench_chain.py needs an H100: the magnification core has no CPU fallback")
    lanes, T = args.lanes, args.clip
    before = card()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=20, wavelength=50.0, low=0.4, high=3.0, chroma=50,
                       levels=LEVELS, captureFps=30.0)
    cfg = L.ProcessorConfig(preprocess=L.PreprocessParams(DOWN), magnification=L.toParams(ui))

    # distinct 4K source frames (content does not change the work), tiled over the clip's virtual lanes on the device
    base = [cv2.resize(synth_frame(t, DW, DH, 3), (SW, SH), interpolation=cv2.INTER_LINEAR) for t in range(4)]

    def nv12(f):
        i420, n = cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420).ravel(), SW * SH
        uv = np.stack([i420[n:n + n // 4], i420[n + n // 4:]], -1).reshape(SH // 2, SW)
        return np.concatenate([i420[:n].reshape(SH, SW), uv])

    vl = T * lanes
    lane_nv, row, orow = SW * SH * 3 // 2, SW * 3, DW * 3
    bgr_src = torch.from_numpy(np.stack(base)).cuda()
    nv_src = torch.from_numpy(np.stack([nv12(f) for f in base])).cuda()
    bgr_d = torch.stack([bgr_src[v % 4] for v in range(vl)])
    nv_d = torch.stack([nv_src[v % 4] for v in range(vl)])
    conv_d = torch.empty((vl, SH, SW, 3), dtype=torch.uint8, device="cuda")     # nv12_convert's 4K BGR frames
    out_d = torch.empty((vl, DH, DW, 3), dtype=torch.uint8, device="cuda")
    orig_d = torch.empty_like(out_d)
    torch.cuda.synchronize()
    planes = lambda base_ptr: capi.McNv12(base_ptr, base_ptr + SW * SH, SW, lane_nv)
    convert = capi.lib().mc_debug_nv12_to_bgr
    convert.restype = C.c_int

    chains = {}

    def chain(key):
        if key not in chains:
            chains[key] = L.ProcessingChainB200(0, lanes=lanes)
        return chains[key]

    def path(kind, n):
        ch = chain((kind, n))
        def call(i):
            off = (i % T) * lanes if n == 1 else 0   # frame calls step through the clip's frames, a clip takes them all
            if kind == "nv12_fused":
                flags, _ = ch.process_nv12_device(planes(nv_d[off].data_ptr()), n, SW, SH, cfg, out_d[off].data_ptr(), orow,
                                                  orig_d[off].data_ptr(), orow)
            else:
                if kind == "nv12_convert":
                    assert convert(C.byref(planes(nv_d[off].data_ptr())), SW, SH, lanes * n, C.c_void_p(conv_d[off].data_ptr()),
                                   C.c_size_t(row)) == 0
                    src = conv_d[off]
                else:
                    src = bgr_d[off]
                flags, _ = ch.process_device(src.data_ptr(), n, SW, SH, 3, row, cfg, out_d[off].data_ptr(), orow,
                                             orig_d[off].data_ptr(), orow)
            return flags

        def run(k):
            calls = max(1, T // n)   # the same frames per timed chunk for frame calls and clips
            for i in range(calls):
                call(k * calls + i)
            ch.magnifier.sync()
        return run, call

    kinds = ("nv12_fused", "nv12_convert", "bgr")
    shapes = {"frame": 1, f"clip{T}": T}
    paths = {f"{k}/{s}": path(k, n) for k in kinds for s, n in shapes.items()}
    for run, _ in paths.values():   # warm-up: module load, staging, tap tables, the first frames' state
        run(0)
        run(1)
    rates = {k: [] for k in paths}
    for _ in range(args.repeats):
        for k, (run, _) in paths.items():
            n, dt = timed(run, args.window)
            rates[k].append(n * T * lanes / dt)
    fps = {k: statistics.median(v) for k, v in rates.items()}

    # device time of the front kernel (profile_kernels) and of the 4K conversion (CUDA events), a pass of their own
    front_us = {}
    for k, (_, call) in paths.items():
        ch = chain((k.split("/")[0], shapes[k.split("/")[1]]))
        ch.magnifier.set_option("profile_kernels", 1)
        ch.magnifier.profile_read()
        calls = 8
        for i in range(calls):
            call(i)
        prof = ch.magnifier.profile_read()
        ch.magnifier.set_option("profile_kernels", 0)
        n_launch, ms = prof[("chain_front", 0)]
        front_us[k] = 1e3 * ms / (n_launch * lanes * shapes[k.split("/")[1]])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    reps = 4
    for _ in range(reps):
        convert(C.byref(planes(nv_d[0].data_ptr())), SW, SH, vl, C.c_void_p(conv_d[0].data_ptr()), C.c_size_t(row))
    ev1.record()
    torch.cuda.synchronize()
    convert_us = 1e3 * ev0.elapsed_time(ev1) / (reps * vl)

    nv_b, bgr_b, out_b = SW * SH * 1.5, SW * SH * 3.0, DW * DH * 3.0
    counted = {"nv12_fused": nv_b + out_b, "nv12_convert": bgr_b + out_b, "bgr": bgr_b + out_b}
    after = card()
    result = {
        "workload": f"{SW}x{SH} source, downscale {DOWN} -> {DW}x{DH} Laplace, {LEVELS} levels, {lanes} lanes, "
                    f"frame calls and clips of {T}, original tap written",
        "frames_per_s": {k: round(v, 1) for k, v in fps.items()},
        "chain_front_us_per_frame": {k: round(v, 3) for k, v in front_us.items()},
        "chain_front_bytes_per_frame": {k: counted[k.split("/")[0]] for k in paths},
        "chain_front_share_of_3.35TBps": {k: round(counted[k.split("/")[0]] / PEAK * 1e6 / v, 3) for k, v in front_us.items()},
        "nv12_to_bgr_4k_us_per_frame": round(convert_us, 3),
        "nv12_to_bgr_4k_bytes_per_frame": nv_b + bgr_b,
        "nv12_to_bgr_4k_share_of_3.35TBps": round((nv_b + bgr_b) / PEAK * 1e6 / convert_us, 3),
        "window_s": args.window, "repeats": args.repeats,
        "card_before": before, "card_after": after,
    }
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')})", flush=True)
    print(json.dumps(result), flush=True)
    for c in chains.values():
        c.magnifier.close()


if __name__ == "__main__":
    main()
