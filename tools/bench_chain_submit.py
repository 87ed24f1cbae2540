#!/usr/bin/env python
"""Host frames through the processing chain: the pipelined chain submits (mc_chain_submit / mc_chain_submit_yuv422,
pipeline_depth 3, submit frame N+1 before collecting frame N) against what a caller does without them, in frames/s:
  - 1 lane: a loop of the blocking mc_chain_process / mc_chain_process_yuv422;
  - 16 and 64 lanes: the caller's own async copies on the handle's stream + mc_chain_process_device + a synchronise per
    step.
1080p BGR or YUYV host frames, pinned, at bench.py's Laplace parameters (6 levels), downscale 1 and 2, no original tap
requested.  Each leg is warmed up, then timed over windows of at least `--window` seconds (median of `--repeats`, legs
alternating).  Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

    python tools/bench_chain_submit.py [--window 2.0] [--repeats 3] [--lanes 1,16,64]"""
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

from bench_nv12 import card  # noqa: E402

W, H, DEPTH = 1920, 1080, 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lanes", default="1,16,64")
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.processor import _to_mc
    from lvm_b200.synth import synth_frame
    from bench import UI

    if not torch.cuda.is_available():
        raise SystemExit("bench_chain_submit.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    lib = capi.lib()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=UI["amplification"], wavelength=UI["wavelength"],
                       low=UI["low"], high=UI["high"], chroma=UI["chroma"], levels=UI["levels"], captureFps=UI["fps"])

    def cfg_of(down):
        return L.ProcessorConfig(magnification=L.toParams(ui), preprocess=L.PreprocessParams(down))

    bgr = synth_frame(0, W, H, 3, seed=1)
    ycc = cv2.cvtColor(bgr, cv2.COLOR_BGR2YCrCb)
    y = ycc[..., 0].reshape(H, W // 2, 2)
    yuyv = np.stack([y[..., 0], ycc[:, ::2, 2], y[..., 1], ycc[:, ::2, 1]], -1).reshape(H, 2 * W)

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8).pin_memory()

    def leg(kind, down, lanes):
        """-> {name: step function that moves one frame of every lane}, and what to keep alive"""
        cfg = cfg_of(down)
        p = _to_mc(cfg)
        row_in = 3 * W if kind == "bgr" else 2 * W
        h_in = pinned(lanes * H * row_in)
        h_in.view(lanes, H, row_in).copy_(torch.from_numpy(bgr.reshape(H, -1) if kind == "bgr" else yuyv))
        g = L.ProcessingChainB200.geometry(cfg, W, H, 3)
        ow, oh = (W, H) if g.cur_is_input else (g.out_w, g.out_h)
        out_row = 3 * ow
        outs = [pinned(lanes * oh * out_row) for _ in range(DEPTH)]
        yv = capi.McYuv422(h_in.data_ptr(), row_in, row_in * H, capi.MC_YUV422_YUYV)
        steps = {}

        # the chain submits: submit frame N+1, then collect frame N
        sub = L.ProcessingChainB200(0, lanes=lanes)
        sub.magnifier.set_option("pipeline_depth", DEPTH)
        state = dict(n=0, inflight=0)

        def submit_step(k):
            if state["inflight"] == DEPTH:
                sub.collect()
                state["inflight"] -= 1
            out = outs[k % DEPTH].data_ptr()
            if kind == "bgr":
                sub.submit(h_in.data_ptr(), W, H, 3, row_in, cfg, out, out_row)
            else:
                sub.submit_yuv422(yv, W, H, cfg, out, out_row)
            state["inflight"] += 1

        def drain():
            while state["inflight"]:
                sub.collect()
                state["inflight"] -= 1

        steps["submit"] = (submit_step, drain)

        if lanes == 1:   # the blocking host call
            blk = L.ProcessingChainB200(0)
            info = capi.McChainInfo()
            out = outs[0]

            def blocking_step(k):
                if kind == "bgr":
                    st = lib.mc_chain_process(blk.magnifier._h, h_in.data_ptr(), W, H, 3, row_in, C.byref(p), 0, out.data_ptr(),
                                              out.numel(), None, 0, C.byref(info))
                else:
                    st = lib.mc_chain_process_yuv422(blk.magnifier._h, C.byref(yv), W, H, C.byref(p), 0, out.data_ptr(),
                                                     out.numel(), None, 0, C.byref(info))
                assert st == capi.MC_OK

            steps["blocking"] = (blocking_step, lambda: None)
        else:            # the caller's own copies + the device chain call + a synchronise per step
            dev = L.ProcessingChainB200(0, lanes=lanes)
            d_in = torch.empty(h_in.numel(), dtype=torch.uint8, device="cuda")
            d_out = torch.empty(outs[0].numel(), dtype=torch.uint8, device="cuda")
            stream = torch.cuda.ExternalStream(dev.magnifier.stream)
            dyv = capi.McYuv422(d_in.data_ptr(), row_in, row_in * H, capi.MC_YUV422_YUYV)

            def device_step(k):
                with torch.cuda.stream(stream):
                    d_in.copy_(h_in, non_blocking=True)
                    if kind == "bgr":
                        dev.process_device(d_in.data_ptr(), 1, W, H, 3, row_in, cfg, d_out.data_ptr(), out_row)
                    else:
                        dev.process_yuv422_device(dyv, 1, W, H, cfg, d_out.data_ptr(), out_row)
                    outs[0].copy_(d_out, non_blocking=True)
                stream.synchronize()

            steps["device_call"] = (device_step, lambda: None)
        return steps

    def rate(step, finish, lanes, window):
        t0, n = time.perf_counter(), 0
        while time.perf_counter() - t0 < window:
            step(n)
            n += 1
        finish()
        return n * lanes / (time.perf_counter() - t0)

    results = []
    for lanes in [int(x) for x in args.lanes.split(",")]:
        for kind in ("bgr", "yuyv"):
            for down in (1, 2):
                steps = leg(kind, down, lanes)
                for step, finish in steps.values():   # warm-up: every shape, the slots, the tap tables
                    for k in range(10):
                        step(k)
                    finish()
                runs = {name: [] for name in steps}
                for _ in range(args.repeats):
                    for name, (step, finish) in steps.items():
                        runs[name].append(rate(step, finish, lanes, args.window))
                r = dict(source=kind, downscale=down, lanes=lanes,
                         **{f"{name}_fps": round(statistics.median(v), 1) for name, v in runs.items()},
                         spread={name: [round(x, 1) for x in v] for name, v in runs.items()})
                print(r, flush=True)
                results.append(r)
                del steps
                torch.cuda.synchronize()
    after = card()
    print("card before:", before)
    print("card after: ", after)
    print(json.dumps(dict(card=before, window_s=args.window, repeats=args.repeats, depth=DEPTH, results=results)))


if __name__ == "__main__":
    main()
