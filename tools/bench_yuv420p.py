#!/usr/bin/env python
"""A software exporter's loop on I420 frames: 1 lane of 1080p I420 host frames (what FFmpeg's software decoders hand out)
at bench.py's Laplace parameters (6 levels), clips of T = 16, MC_SPLIT_LEFT_RIGHT, into I420 canvases (what libx264 /
FFV1 / MJPEG take), pinned host buffers, pipeline_depth 3.  Legs, alternated in one process:
  (a) mc_chain_compose_submit_yuv420p: I420 frames in, I420 canvases out;
  (b) the NV12 calls: the host interleaves each frame's chroma before mc_chain_compose_submit_nv12 and de-interleaves
      each NV12 canvas after collect (numpy);
  (c) the BGR route: the host converts each frame with cv2.cvtColor(YUV2BGR_I420) before mc_chain_compose_submit, and
      each BGR canvas with cvtColor(BGR2YUV_I420) after collect;
  (d) the copy ceiling of (a)'s bytes: the I420 clip up and its I420 canvases down, pinned, on two streams, no kernel.
Reports canvases per second and the calling thread's CPU time per canvas (time.thread_time), each the median of
`--repeats` windows of at least `--window` seconds, with the card's name, power limit and SM clocks read in the same run,
and one JSON line.  No labels are drawn.

    python tools/bench_yuv420p.py [--window 2.0] [--repeats 3] [--legs a,b,c,d]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_nv12 import card  # noqa: E402

W, H, T, DEPTH = 1920, 1080, 16, 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--legs", default="a,b,c,d")
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.synth import synth_frame
    from bench import UI

    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv420p.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=UI["amplification"], wavelength=UI["wavelength"],
                       low=UI["low"], high=UI["high"], chroma=UI["chroma"], levels=UI["levels"], captureFps=UI["fps"])
    cfg = L.ProcessorConfig(magnification=L.toParams(ui))
    split = capi.MC_SPLIT_LEFT_RIGHT
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, split)
    fb, cb = W * H * 3 // 2, cw * ch * 3 // 2           # I420 bytes of a frame and of a canvas
    i420 = [cv2.cvtColor(synth_frame(t, W, H, 3, seed=1), cv2.COLOR_BGR2YUV_I420) for t in range(2)]

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8).pin_memory()

    def np_of(t, shape):
        return t.numpy().reshape(shape)

    def i420_clip():
        buf = pinned(T * fb)
        a = np_of(buf, (T, H * 3 // 2, W))
        for t in range(T):
            a[t] = i420[t % 2]
        return buf

    def planes(base, w, h, lanes_bytes):
        return capi.McYuv420p(base, base + w * h, base + w * h + (w // 2) * (h // 2), w, w // 2, lanes_bytes)

    def canvas_of(fmt, base):
        if fmt == capi.MC_CANVAS_BGR:
            return capi.McCanvas(fmt, base, None, 3 * cw, 3 * cw * ch)
        return capi.McCanvas(fmt, base, base + cw * ch, cw, cb)

    def pipeline(submit, post):
        """-> (step, drain): step(k) collects the oldest clip when DEPTH are in flight (then post(slot) on its canvases)
        and submits clip k into slot k % DEPTH"""
        state = dict(inflight=[])

        def step(k):
            if len(state["inflight"]) == DEPTH:
                sub.magnifier.collect()
                post(state["inflight"].pop(0))
            submit(k % DEPTH)
            state["inflight"].append(k % DEPTH)

        def drain():
            while state["inflight"]:
                sub.magnifier.collect()
                post(state["inflight"].pop(0))

        sub = L.ProcessingChainB200(0)
        sub.magnifier.set_option("pipeline_depth", DEPTH)
        return step, drain, sub

    def leg_i420():
        """(a): I420 in, I420 canvases out"""
        h_in = i420_clip()
        outs = [pinned(T * cb) for _ in range(DEPTH)]

        def submit(s):
            chain.compose_submit_yuv420p(planes(h_in.data_ptr(), W, H, fb), T, W, H, cfg, split,
                                         canvas_of(capi.MC_CANVAS_I420, outs[s].data_ptr()))

        step, drain, chain = pipeline(submit, lambda s: None)
        return step, drain, (h_in, outs, chain)

    def leg_nv12():
        """(b): interleave before the NV12 submit, de-interleave after collect"""
        src = np_of(i420_clip(), (T, H * 3 // 2 * W))
        ins = [pinned(T * fb) for _ in range(DEPTH)]
        outs = [pinned(T * cb) for _ in range(DEPTH)]
        final = np.empty((T, cb), np.uint8)
        n, q = W * H, W * H // 4
        cn, cq = cw * ch, cw * ch // 4

        def submit(s):
            a = np_of(ins[s], (T, fb))
            a[:, :n] = src[:, :n]
            uv = a[:, n:].reshape(T, q, 2)
            uv[..., 0] = src[:, n:n + q]
            uv[..., 1] = src[:, n + q:]
            base = ins[s].data_ptr()
            chain.compose_submit_nv12(capi.McNv12(base, base + n, W, fb), T, W, H, cfg, split,
                                      canvas_of(capi.MC_CANVAS_NV12, outs[s].data_ptr()))

        def post(s):
            c = np_of(outs[s], (T, cb))
            final[:, :cn] = c[:, :cn]
            uv = c[:, cn:].reshape(T, cq, 2)
            final[:, cn:cn + cq] = uv[..., 0]
            final[:, cn + cq:] = uv[..., 1]

        step, drain, chain = pipeline(submit, post)
        return step, drain, (ins, outs, chain)

    def leg_bgr():
        """(c): cv2 YUV2BGR_I420 before the BGR submit, BGR2YUV_I420 after collect"""
        src = np_of(i420_clip(), (T, H * 3 // 2, W))
        ins = [pinned(T * W * H * 3) for _ in range(DEPTH)]
        outs = [pinned(T * 3 * cw * ch) for _ in range(DEPTH)]
        final = np.empty((T, ch * 3 // 2, cw), np.uint8)

        def submit(s):
            a = np_of(ins[s], (T, H, W, 3))
            for t in range(T):
                cv2.cvtColor(src[t], cv2.COLOR_YUV2BGR_I420, dst=a[t])
            chain.compose_submit(ins[s].data_ptr(), T, W, H, 3, 3 * W, cfg, split, canvas_of(capi.MC_CANVAS_BGR, outs[s].data_ptr()))

        def post(s):
            c = np_of(outs[s], (T, ch, cw, 3))
            for t in range(T):
                cv2.cvtColor(c[t], cv2.COLOR_BGR2YUV_I420, dst=final[t])

        step, drain, chain = pipeline(submit, post)
        return step, drain, (ins, outs, chain)

    def leg_copies():
        """(d): (a)'s bytes each way on two streams, pinned, no kernel"""
        h_in = pinned(T * fb)
        h_out = [pinned(T * cb) for _ in range(DEPTH)]
        d_in = [torch.empty(T * fb, dtype=torch.uint8, device="cuda") for _ in range(DEPTH)]
        d_out = [torch.empty(T * cb, dtype=torch.uint8, device="cuda") for _ in range(DEPTH)]
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

        return step, torch.cuda.synchronize, (h_in, h_out, d_in, d_out)

    makers = {"a": ("a_i420_in_i420_canvas", leg_i420), "b": ("b_nv12_calls_host_repack", leg_nv12),
              "c": ("c_bgr_calls_host_cvtcolor", leg_bgr), "d": ("d_copy_ceiling_i420", leg_copies)}
    built = {}
    for key in args.legs.split(","):
        name, make = makers[key]
        step, drain, keep = make()
        for k in range(2 * DEPTH + 2):   # warm-up: the slots, the staging, the clip scratch
            step(k)
        drain()
        built[name] = (step, drain, keep)

    def rate(step, drain, window):
        t0, c0, n = time.perf_counter(), time.thread_time(), 0
        while time.perf_counter() - t0 < window:
            step(n)
            n += 1
        drain()
        return n * T / (time.perf_counter() - t0), (time.thread_time() - c0) * 1e3 / (n * T)

    runs = {name: [] for name in built}
    for _ in range(args.repeats):
        for name, (step, drain, _) in built.items():
            runs[name].append(rate(step, drain, args.window))
    results = {name: dict(canvases_per_s=round(statistics.median(r for r, _ in v), 1),
                          host_cpu_ms_per_canvas=round(statistics.median(c for _, c in v), 3),
                          spread=[round(r, 1) for r, _ in v]) for name, v in runs.items()}
    for name, r in results.items():
        print(f"{name:32s} {r['canvases_per_s']:9.1f} canvases/s  {r['host_cpu_ms_per_canvas']:7.3f} host CPU ms/canvas  "
              f"{r['spread']}", flush=True)
    after = card()
    print("card before:", before)
    print("card after: ", after)
    print(json.dumps(dict(card=before, window_s=args.window, repeats=args.repeats, depth=DEPTH, clip=T, canvas=[cw, ch],
                          bytes_per_canvas=dict(up=fb, down=cb), results=results)))


if __name__ == "__main__":
    main()
