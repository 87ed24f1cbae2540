#!/usr/bin/env python
"""Packed 4:2:2 camera frames (YUYV) against BGR frames into the processing chain, in one process that alternates the
paths in windows of at least `--window` seconds (median of `--repeats`):
  1. the host's cv2.cvtColor(COLOR_YUV2BGR_YUYV) per 1080p frame on 1 thread and on all threads: the CPU work that a
     camera source pays today and that mc_chain_process_yuv422 removes;
  2. the blocking 1-lane 1080p chain call (Laplace, no front stage), mc_chain_process_yuv422 against mc_chain_process,
     with pinned and with pageable host frames (ms per frame); the 4:2:2 call also with `original` NULL, since it
     otherwise downloads the converted original frame that a BGR caller already holds;
  3. the chain_front kernel's device time per frame (profile_kernels) for a YUYV and a BGR source, 1080p copy and 4K ->
     1080p downscale 2, and its share of the byte floor (bytes read + written at the data-sheet 3.35 TB/s);
  4. 16 lanes of device-resident 1080p Laplace chain calls, mc_chain_process_yuv422_device against
     mc_chain_process_device (frames/s).
Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

    python tools/bench_yuv422.py [--window 1.0] [--repeats 3]"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card, timed  # noqa: E402

W, H, LEVELS = 1920, 1080, 6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lanes", type=int, default=16)
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.processor import _to_mc
    from lvm_b200.synth import synth_frame

    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv422.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=20, wavelength=50.0, low=0.4, high=3.0, chroma=50,
                       levels=LEVELS, captureFps=30.0)
    cfg = L.ProcessorConfig(magnification=L.toParams(ui))
    p = _to_mc(cfg)
    lib = capi.lib()

    def yuyv(bgr):
        """BGR -> YUYV [h][2w] (luma and each pair's left chroma; content does not change the work)"""
        ycc = cv2.cvtColor(bgr, cv2.COLOR_BGR2YCrCb)
        h, w = bgr.shape[:2]
        y = ycc[..., 0].reshape(h, w // 2, 2)
        return np.stack([y[..., 0], ycc[:, ::2, 2], y[..., 1], ycc[:, ::2, 1]], -1).reshape(h, 2 * w)

    T = 4
    frames = [synth_frame(t, W, H, 3) for t in range(T)]
    yu = [yuyv(f) for f in frames]
    result = {}

    def median_rate(fns, unit):
        """fns: name -> run(k); alternated, median of repeats -> name -> calls per second"""
        for fn in fns.values():
            fn(0)
        r = {k: [] for k in fns}
        for _ in range(args.repeats):
            for k, fn in fns.items():
                n, dt = timed(fn, args.window)
                r[k].append(n * unit / dt)
        return {k: statistics.median(v) for k, v in r.items()}

    # 1. the host conversion
    threads = cv2.getNumThreads()
    conv = {}
    for nt in (1, threads):
        cv2.setNumThreads(nt)
        conv[nt] = median_rate({"cvt": lambda k: [cv2.cvtColor(yu[i].reshape(H, W, 2), cv2.COLOR_YUV2BGR_YUYV)
                                                  for i in range(T)]}, T)["cvt"]
    cv2.setNumThreads(threads)
    result["host_cvtcolor_ms_per_frame"] = {"1_thread": round(1e3 / conv[1], 3), f"{threads}_threads": round(1e3 / conv[threads], 3)}

    # 2. the blocking 1-lane host call
    ch_y, ch_b = L.ProcessingChainB200(0), L.ProcessingChainB200(0)
    out, orig = np.empty(W * H * 3, np.uint8), np.empty(W * H * 3, np.uint8)
    info = capi.McChainInfo()

    def host_frames(pinned):
        if not pinned:
            return [np.ascontiguousarray(f) for f in frames], [np.ascontiguousarray(f) for f in yu]
        return ([torch.from_numpy(f).pin_memory().numpy() for f in frames], [torch.from_numpy(f).pin_memory().numpy() for f in yu])

    host = {}
    for pinned in (False, True):
        bf, yf = host_frames(pinned)
        tag = "pinned" if pinned else "pageable"

        def run_y(k, yf=yf, with_orig=True):
            for i in range(T):
                yv = capi.McYuv422(yf[i].ctypes.data, 2 * W, 0, capi.MC_YUV422_YUYV)
                assert lib.mc_chain_process_yuv422(ch_y.magnifier._h, C.byref(yv), W, H, C.byref(p), 0, out.ctypes.data,
                                                   out.size, orig.ctypes.data if with_orig else None, orig.size,
                                                   C.byref(info)) == 0

        def run_b(k, bf=bf):
            for i in range(T):
                assert lib.mc_chain_process(ch_b.magnifier._h, bf[i].ctypes.data, W, H, 3, 3 * W, C.byref(p), 0,
                                            out.ctypes.data, out.size, orig.ctypes.data, orig.size, C.byref(info)) == 0

        # yuyv downloads the converted original too (the BGR call's original is the caller's own input frame)
        r = median_rate({"yuyv": run_y, "yuyv_no_original": lambda k: run_y(k, with_orig=False), "bgr": run_b}, T)
        host[tag] = {k: round(1e3 / v, 3) for k, v in r.items()}
    result["blocking_1lane_ms_per_frame"] = host

    # 3. chain_front device time, and 4. 16 device lanes
    lanes = args.lanes
    SW, SH = 2 * W, 2 * H
    big = [cv2.resize(f, (SW, SH), interpolation=cv2.INTER_LINEAR) for f in frames]
    src = {
        "copy_1080p": (W, H, frames, yu, 1),
        "down2_4k": (SW, SH, big, [yuyv(f) for f in big], 2),
    }
    front = {}
    for name, (w, h, bgr, yy, down) in src.items():
        fcfg = L.ProcessorConfig(preprocess=L.PreprocessParams(down), magnification=L.toParams(
            L.MagUiValues(mode=L.MagnificationMode.NONE)))
        bgr_d = torch.from_numpy(np.stack([bgr[v % T] for v in range(lanes)])).cuda()
        y_d = torch.from_numpy(np.stack([yy[v % T] for v in range(lanes)])).cuda()
        dw, dh = w // down, h // down
        out_d, orig_d = (torch.empty((lanes, dh, dw, 3), dtype=torch.uint8, device="cuda") for _ in range(2))
        ch = L.ProcessingChainB200(0, lanes=lanes)
        ch.magnifier.set_option("profile_kernels", 1)
        us = {}
        for kind in ("yuyv", "bgr"):
            def call():
                if kind == "yuyv":
                    ch.process_yuv422_device(capi.McYuv422(y_d.data_ptr(), 2 * w, 2 * w * h, capi.MC_YUV422_YUYV), 1, w, h, fcfg,
                                             out_d.data_ptr(), 3 * dw, orig_d.data_ptr() if down == 1 else 0, 3 * dw)
                else:   # the BGR front with a Preprocess stage writes its output once, into d_original
                    ch.process_device(bgr_d.data_ptr(), 1, w, h, 3, 3 * w, fcfg, out_d.data_ptr(), 3 * dw, orig_d.data_ptr(),
                                      3 * dw)
            for _ in range(3):
                call()
            ch.magnifier.sync()
            ch.magnifier.profile_read()
            n = 50
            for _ in range(n):
                call()
            ch.magnifier.sync()
            prof = ch.magnifier.profile_read()
            launches, ms = prof.get(("chain_front", 0), (0, 0.0))
            us[kind] = 1e3 * ms / max(launches, 1) / lanes
        in_b = {"yuyv": 2 * w * h, "bgr": 3 * w * h}
        out_b = 3 * dw * dh
        front[name] = {k: {"us_per_frame": round(v, 3), "bytes": in_b[k] + out_b,
                           "share_of_floor": round((in_b[k] + out_b) / 3.35e12 * 1e6 / v, 3) if v > 0 else None}
                       for k, v in us.items()}
        if down == 1:   # a BGR source without a front stage launches none: its front time is 0 (the magnifier reads d_in)
            front[name]["bgr"]["note"] = "no front launch for a BGR source without a front stage"
        ch.magnifier.close()
    result["chain_front"] = front

    bgr_d = torch.from_numpy(np.stack([frames[v % T] for v in range(lanes)])).cuda()
    y_d = torch.from_numpy(np.stack([yu[v % T] for v in range(lanes)])).cuda()
    out_d = torch.empty((lanes, H, W, 3), dtype=torch.uint8, device="cuda")
    chy, chb = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)
    steps = 8

    def dev(kind):
        def run(k):
            for _ in range(steps):
                if kind == "yuyv":
                    chy.process_yuv422_device(capi.McYuv422(y_d.data_ptr(), 2 * W, 2 * W * H, capi.MC_YUV422_YUYV), 1, W, H, cfg,
                                              out_d.data_ptr(), 3 * W)
                else:
                    chb.process_device(bgr_d.data_ptr(), 1, W, H, 3, 3 * W, cfg, out_d.data_ptr(), 3 * W)
            (chy if kind == "yuyv" else chb).magnifier.sync()
        return run

    result["device_16lane_frames_per_s"] = {k: round(v, 1) for k, v in
                                             median_rate({"yuyv": dev("yuyv"), "bgr": dev("bgr")}, steps * lanes).items()}
    result.update(workload=f"Laplace {W}x{H}, {LEVELS} levels, chroma 50", window_s=args.window, repeats=args.repeats,
                  card_before=before, card_after=card())
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')})", flush=True)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
