#!/usr/bin/env python
"""RGB frames into the chain, at bench.py's Laplace parameters (6 levels), clips of T = 16, MC_SPLIT_LEFT_RIGHT.  Legs,
alternated in one process:
  device (16 lanes of 1080p planar RGB, (N, 3, H, W) CUDA tensors, into NV12 canvases; frames per second):
    (a) mc_chain_compose_rgb_device on the tensor's planes;
    (b) torch's flip(0).permute(1, 2, 0) of every frame into one HWC BGR buffer (a single copy_ over the clip, on the
        handle's stream), then mc_chain_compose_device;
  host (the exporter's loop: 1 lane of pinned 1080p host frames, pipeline_depth 3, RGB canvases; canvases per second and
  the calling thread's CPU ms per canvas):
    (c) mc_chain_compose_submit_rgb on rgb24 frames;   (d) the same on BGRA frames;
    (e) cv2.cvtColor(RGB2BGR) of each rgb24 frame on the calling thread, mc_chain_compose_submit, BGR canvases, and
        cv2.cvtColor(BGR2RGB) of each canvas after collect;   (f) the same from BGRA frames (BGRA2BGR);
    (g) the copy ceiling of (c)'s bytes: the rgb24 clip up and its RGB canvases down, pinned, on two streams, no kernel.
Each figure is the median of `--repeats` windows of at least `--window` seconds, with the card's name, power limit and
SM clocks read in the same run, and one JSON line.  No labels are drawn.

    python tools/bench_rgb.py [--window 2.0] [--repeats 3] [--legs a,b,c,d,e,f,g]"""
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

W, H, T, DEPTH, DEV_LANES = 1920, 1080, 16, 3, 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--legs", default="a,b,c,d,e,f,g")
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.synth import synth_frame
    from bench import UI

    if not torch.cuda.is_available():
        raise SystemExit("bench_rgb.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    ui = L.MagUiValues(mode=L.MagnificationMode.Laplace, amplification=UI["amplification"], wavelength=UI["wavelength"],
                       low=UI["low"], high=UI["high"], chroma=UI["chroma"], levels=UI["levels"], captureFps=UI["fps"])
    cfg = L.ProcessorConfig(magnification=L.toParams(ui))
    split = capi.MC_SPLIT_LEFT_RIGHT
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, split)
    bgr = [synth_frame(t, W, H, 3, seed=1) for t in range(2)]
    rgb24 = [cv2.cvtColor(f, cv2.COLOR_BGR2RGB) for f in bgr]
    bgra = [cv2.cvtColor(f, cv2.COLOR_BGR2BGRA) for f in bgr]

    def pinned(nbytes):
        return torch.empty(nbytes, dtype=torch.uint8).pin_memory()

    def np_of(t, shape):
        return t.numpy().reshape(shape)

    # ---- device legs: an (N, 3, H, W) tensor of every lane's clip, N = T * DEV_LANES (virtual lane t * lanes + k)
    def device_leg(native):
        chain = L.ProcessingChainB200(0, lanes=DEV_LANES)
        m = chain.magnifier
        n = T * DEV_LANES
        x = torch.stack([torch.from_numpy(rgb24[i % 2]).permute(2, 0, 1) for i in range(n)]).cuda()   # (N, 3, H, W)
        nv_bytes = cw * ch * 3 // 2
        canvases = torch.empty(n * nv_bytes, dtype=torch.uint8, device="cuda")
        canvas = capi.McCanvas(capi.MC_CANVAS_NV12, canvases.data_ptr(), canvases.data_ptr() + cw * ch, cw, nv_bytes)
        stream = torch.cuda.ExternalStream(m.stream)
        hwc = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
        plane = H * W

        def step(k):
            if native:
                base = x.data_ptr()
                m.chain_compose_rgb_device(capi.McRgb(base, base + plane, base + 2 * plane, W, 3 * plane, capi.MC_RGB_PLANAR),
                                           T, W, H, cfg, split, canvas)
            else:
                with torch.cuda.stream(stream):   # ordered before the compose on the handle's stream; one pass over the clip
                    hwc.copy_(x.flip(1).permute(0, 2, 3, 1))
                m.chain_compose_device(hwc.data_ptr(), T, W, H, 3, 3 * W, cfg, split, canvas)

        return step, m.sync, (chain, x, canvases, hwc), n

    # ---- host legs
    def pipeline(submit, post):
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

    def host_clip(frames, bpp):
        buf = pinned(T * W * H * bpp)
        a = np_of(buf, (T, H, W, bpp))
        for t in range(T):
            a[t] = frames[t % 2]
        return buf

    def canvas_of(fmt, base):
        return capi.McCanvas(fmt, base, None, 3 * cw, 3 * cw * ch)

    def native_host_leg(frames, bpp, layout):
        h_in = host_clip(frames, bpp)
        outs = [pinned(T * 3 * cw * ch) for _ in range(DEPTH)]

        def submit(s):
            chain.compose_submit_rgb(capi.McRgb(h_in.data_ptr(), None, None, bpp * W, bpp * W * H, layout), T, W, H, cfg, split,
                                     canvas_of(capi.MC_CANVAS_RGB, outs[s].data_ptr()))

        step, drain, chain = pipeline(submit, lambda s: None)
        return step, drain, (h_in, outs, chain), T

    def cvt_host_leg(frames, bpp, code):
        src = np_of(host_clip(frames, bpp), (T, H, W, bpp))
        ins = [pinned(T * W * H * 3) for _ in range(DEPTH)]
        outs = [pinned(T * 3 * cw * ch) for _ in range(DEPTH)]
        final = np.empty((T, ch, cw, 3), np.uint8)

        def submit(s):
            a = np_of(ins[s], (T, H, W, 3))
            for t in range(T):
                cv2.cvtColor(src[t], code, dst=a[t])
            chain.compose_submit(ins[s].data_ptr(), T, W, H, 3, 3 * W, cfg, split, canvas_of(capi.MC_CANVAS_BGR, outs[s].data_ptr()))

        def post(s):
            c = np_of(outs[s], (T, ch, cw, 3))
            for t in range(T):
                cv2.cvtColor(c[t], cv2.COLOR_BGR2RGB, dst=final[t])

        step, drain, chain = pipeline(submit, post)
        return step, drain, (ins, outs, chain), T

    def copies_leg():
        fb, cb = W * H * 3, 3 * cw * ch
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

        return step, torch.cuda.synchronize, (h_in, h_out, d_in, d_out), T

    makers = {"a": ("a_device_planar_rgb", lambda: device_leg(True)),
              "b": ("b_device_torch_permute_then_bgr", lambda: device_leg(False)),
              "c": ("c_host_rgb24", lambda: native_host_leg(rgb24, 3, capi.MC_RGB_RGB)),
              "d": ("d_host_bgra", lambda: native_host_leg(bgra, 4, capi.MC_RGB_BGRA)),
              "e": ("e_host_cvtcolor_rgb24_then_bgr", lambda: cvt_host_leg(rgb24, 3, cv2.COLOR_RGB2BGR)),
              "f": ("f_host_cvtcolor_bgra_then_bgr", lambda: cvt_host_leg(bgra, 4, cv2.COLOR_BGRA2BGR)),
              "g": ("g_copy_ceiling_rgb24", copies_leg)}
    built = {}
    for key in args.legs.split(","):
        name, make = makers[key]
        step, drain, keep, per_step = make()
        for k in range(2 * DEPTH + 2):   # warm-up: the slots, the staging, the clip scratch
            step(k)
        drain()
        built[name] = (step, drain, keep, per_step)

    def rate(step, drain, per_step, window):
        t0, c0, n = time.perf_counter(), time.thread_time(), 0
        while time.perf_counter() - t0 < window:
            step(n)
            n += 1
        drain()
        return n * per_step / (time.perf_counter() - t0), (time.thread_time() - c0) * 1e3 / (n * per_step)

    runs = {name: [] for name in built}
    for _ in range(args.repeats):
        for name, (step, drain, _, per_step) in built.items():
            runs[name].append(rate(step, drain, per_step, args.window))
    results = {name: dict(per_s=round(statistics.median(r for r, _ in v), 1),
                          host_cpu_ms_each=round(statistics.median(c for _, c in v), 3),
                          spread=[round(r, 1) for r, _ in v]) for name, v in runs.items()}
    for name, r in results.items():
        unit = "frames/s  " if name.startswith(("a_", "b_")) else "canvases/s"
        print(f"{name:34s} {r['per_s']:9.1f} {unit} {r['host_cpu_ms_each']:7.3f} host CPU ms each  {r['spread']}", flush=True)
    after = card()
    print("card before:", before)
    print("card after: ", after)
    print(json.dumps(dict(card=before, window_s=args.window, repeats=args.repeats, depth=DEPTH, clip=T, device_lanes=DEV_LANES,
                          canvas=[cw, ch], bytes_per_canvas=dict(up_rgb24=W * H * 3, up_bgra=W * H * 4, down=3 * cw * ch),
                          results=results)))


if __name__ == "__main__":
    main()
