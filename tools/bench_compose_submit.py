#!/usr/bin/env python
"""The exporter's loop from host frames: 1 lane of 1080p BGR host frames at bench.py's Laplace parameters (6 levels),
MC_SPLIT_LEFT_RIGHT, in canvases per second.  Legs, alternated in one process:
  (a) compose submits (mc_chain_compose_submit, pipeline_depth 3, clip N collected before clip N + 3 is submitted), clips
      of T = 1, 4 and 16, BGR and NV12 canvases, pinned and pageable buffers;
  (b) chain submits (mc_chain_submit, depth 3) and the canvas built on the CPU with cv2, as tests/compose_oracle.py
      builds it;
  (c) blocking mc_process_clip on clips of 16 and the CPU canvas;
  (d) the copy ceiling: the same bytes per canvas (the BGR frame up, the canvas down) between pinned host memory and the
      GPU on two streams, with no kernel.
Each leg is warmed up, then timed over windows of at least `--window` seconds (median of `--repeats`).  Prints the
card's name, power limit and SM clocks read in the same run, and one JSON line.  No labels are drawn (the exporter's
textOverlay off).

    python tools/bench_compose_submit.py [--window 2.0] [--repeats 3] [--legs a,b,c,d] [--profile DIR]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_nv12 import card  # noqa: E402

W, H, DEPTH = 1920, 1080, 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--legs", default="a,b,c,d")
    ap.add_argument("--profile", default="", help="write a torch.profiler trace of leg (a), T = 16, BGR canvas, pinned, here")
    args = ap.parse_args()

    import ctypes as C
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.processor import _to_mc
    from lvm_b200.synth import synth_frame
    from compose_oracle import compose
    from bench import UI

    if not torch.cuda.is_available():
        raise SystemExit("bench_compose_submit.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    lib = capi.lib()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=UI["amplification"], wavelength=UI["wavelength"],
                       low=UI["low"], high=UI["high"], chroma=UI["chroma"], levels=UI["levels"], captureFps=UI["fps"])
    cfg = L.ProcessorConfig(magnification=L.toParams(ui))
    p = _to_mc(cfg)
    split = capi.MC_SPLIT_LEFT_RIGHT
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, split)
    row = 3 * W
    frame_bytes = H * row
    canvas_bytes = {capi.MC_CANVAS_BGR: 3 * cw * ch, capi.MC_CANVAS_NV12: cw * ch * 3 // 2}
    bgr = [synth_frame(t, W, H, 3, seed=1) for t in range(2)]

    def host(nbytes, pinned):
        if pinned:
            return torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        t = torch.empty(nbytes, dtype=torch.uint8)
        t.fill_(0)   # pageable pages touched before timing
        return t

    def clip_input(T, pinned):
        h_in = host(T * frame_bytes, pinned)
        for t in range(T):
            h_in[t * frame_bytes:(t + 1) * frame_bytes].copy_(torch.from_numpy(bgr[t % 2].reshape(-1)))
        return h_in

    def leg_compose(T, fmt, pinned):
        """(a): -> (step moving one clip, drain, canvases per step)"""
        sub = L.ProcessingChainB200(0)
        sub.magnifier.set_option("pipeline_depth", DEPTH)
        h_in = clip_input(T, pinned)
        nb = canvas_bytes[fmt]
        outs = [host(T * nb, pinned) for _ in range(DEPTH)]
        canvases = []
        for o in outs:
            base = o.data_ptr()
            if fmt == capi.MC_CANVAS_BGR:
                canvases.append(capi.McCanvas(fmt, base, None, 3 * cw, nb))
            else:
                canvases.append(capi.McCanvas(fmt, base, base + cw * ch, cw, nb))
        state = dict(inflight=0)

        def step(k):
            if state["inflight"] == DEPTH:
                sub.magnifier.collect()
                state["inflight"] -= 1
            sub.compose_submit(h_in.data_ptr(), T, W, H, 3, row, cfg, split, canvases[k % DEPTH])
            state["inflight"] += 1

        def drain():
            while state["inflight"]:
                sub.magnifier.collect()
                state["inflight"] -= 1

        return step, drain, T, (sub, h_in, outs)

    def leg_chain_cpu():
        """(b): chain submits at depth 3, each collected frame composed on the CPU while later frames run"""
        sub = L.ProcessingChainB200(0)
        sub.magnifier.set_option("pipeline_depth", DEPTH)
        h_in = clip_input(2, True)
        ins = [h_in[t * frame_bytes:(t + 1) * frame_bytes] for t in range(2)]
        outs = [host(frame_bytes, True) for _ in range(DEPTH)]
        pending = []

        def finish_one():
            sub.magnifier.collect()
            k_in, out = pending.pop(0)
            compose(bgr[k_in], out.numpy().reshape(H, W, 3), split)

        def step(k):
            if len(pending) == DEPTH:
                finish_one()
            sub.submit(ins[k % 2].data_ptr(), W, H, 3, row, cfg, outs[k % DEPTH].data_ptr(), row)
            pending.append((k % 2, outs[k % DEPTH]))

        def drain():
            while pending:
                finish_one()

        return step, drain, 1, (sub, h_in, outs)

    def leg_blocking_clip(T=16):
        """(c): blocking mc_process_clip, then the CPU canvas of every frame"""
        m = L.MagnificationProcessor(0)
        h_in = clip_input(T, True)
        out = host(T * frame_bytes, True)
        flags = np.zeros(T, np.uint8)

        def step(k):
            st = lib.mc_process_clip(m._h, h_in.data_ptr(), T, W, H, 3, row, C.byref(p), out.data_ptr(), row,
                                     flags.ctypes.data_as(C.POINTER(C.c_uint8)))
            assert st == capi.MC_OK
            o = out.numpy().reshape(T, H, W, 3)
            for t in range(T):
                compose(bgr[t % 2], o[t], split)

        return step, lambda: None, T, (m, h_in, out)

    def leg_copies(fmt, T=16):
        """(d): the bytes of T canvases each way on two streams, pinned, no kernel"""
        h_in = host(T * frame_bytes, True)
        h_out = [host(T * canvas_bytes[fmt], True) for _ in range(DEPTH)]
        d_in = [torch.empty(T * frame_bytes, dtype=torch.uint8, device="cuda") for _ in range(DEPTH)]
        d_out = [torch.empty(T * canvas_bytes[fmt], dtype=torch.uint8, device="cuda") for _ in range(DEPTH)]
        s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()
        done = [None] * DEPTH

        def step(k):
            i = k % DEPTH
            if done[i] is not None:
                done[i].synchronize()
            with torch.cuda.stream(s_in):
                d_in[i].copy_(h_in, non_blocking=True)
            with torch.cuda.stream(s_out):
                h_out[i].copy_(d_out[i], non_blocking=True)
                done[i] = torch.cuda.Event()
                done[i].record(s_out)

        def drain():
            torch.cuda.synchronize()

        return step, drain, T, (h_in, h_out, d_in, d_out)

    legs = {}
    want = set(args.legs.split(","))
    if "a" in want:
        for T in (1, 4, 16):
            for fmt, fname in ((capi.MC_CANVAS_BGR, "bgr"), (capi.MC_CANVAS_NV12, "nv12")):
                for pinned in (True, False):
                    legs[f"a_compose_submit_T{T}_{fname}_{'pinned' if pinned else 'pageable'}"] = (leg_compose, (T, fmt, pinned))
    if "b" in want:
        legs["b_chain_submit_cpu_canvas"] = (leg_chain_cpu, ())
    if "c" in want:
        legs["c_blocking_clip16_cpu_canvas"] = (leg_blocking_clip, ())
    if "d" in want:
        legs["d_copy_ceiling_bgr"] = (leg_copies, (capi.MC_CANVAS_BGR,))
        legs["d_copy_ceiling_nv12"] = (leg_copies, (capi.MC_CANVAS_NV12,))

    def rate(step, drain, per_step, window):
        t0, n = time.perf_counter(), 0
        while time.perf_counter() - t0 < window:
            step(n)
            n += 1
        drain()
        return n * per_step / (time.perf_counter() - t0)

    built = {}
    for name, (make, a) in legs.items():   # warm-up: the slots, the staging, the clip scratch
        step, drain, per, keep = make(*a)
        for k in range(2 * DEPTH + 2):
            step(k)
        drain()
        built[name] = (step, drain, per, keep)
    runs = {name: [] for name in legs}
    for _ in range(args.repeats):
        for name, (step, drain, per, _) in built.items():
            runs[name].append(rate(step, drain, per, args.window))
    results = {name: dict(canvases_per_s=round(statistics.median(v), 1), spread=[round(x, 1) for x in v])
               for name, v in runs.items()}
    for name, r in results.items():
        print(f"{name:45s} {r['canvases_per_s']:10.1f}  {r['spread']}", flush=True)

    if args.profile and "a_compose_submit_T16_bgr_pinned" in built:
        from torch.profiler import ProfilerActivity, profile
        step, drain, _, _ = built["a_compose_submit_T16_bgr_pinned"]
        os.makedirs(args.profile, exist_ok=True)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for k in range(12):
                step(k)
            drain()
        prof.export_chrome_trace(os.path.join(args.profile, "compose_submit_T16_bgr_pinned.json"))
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=15), flush=True)

    after = card()
    print("card before:", before)
    print("card after: ", after)
    print(json.dumps(dict(card=before, window_s=args.window, repeats=args.repeats, depth=DEPTH, canvas=[cw, ch],
                          bytes_per_canvas=dict(up=frame_bytes, down_bgr=canvas_bytes[capi.MC_CANVAS_BGR],
                                                down_nv12=canvas_bytes[capi.MC_CANVAS_NV12]), results=results)))


if __name__ == "__main__":
    main()
