#!/usr/bin/env python
"""The export canvas at 1080p: NV12 decoder frames in, Laplace (the bench's settings), the original and processed frames
side by side (MC_SPLIT_LEFT_RIGHT, 3840 x 1080), an NV12 canvas out for the encoder.  Clips of `--frames` frames on 1
and on `--lanes` lanes; one process alternates two paths in windows of at least `--window` seconds, median of
`--repeats`:
  fused     mc_chain_compose_nv12_device: the chain and one compose launch straight into the NV12 canvases;
  separate  what an integrator writes without it: mc_chain_process_nv12_device into BGR frames, the input converted to
            BGR for the original pane (the mc_debug_nv12_to_bgr kernel), a torch cat of the two panes into a BGR canvas,
            and the mc_debug_bgr_to_nv12 kernel into the NV12 canvases.
Then, in a pass of its own, the compose kernel's device time (profile_kernels) and its bytes over that time against the
data-sheet 3.35 TB/s: per canvas it reads 1.5 B/px of NV12 input and 3 B/px of BGR output and writes 1.5 B/px of NV12
over two panes.  Prints the card's name, power limit and SM clocks read in the same run, and one JSON line.

--labels measures the exporter's burnt-in labels instead (mc_set_overlay with lvm_b200.labels.export_labels): on
`--lanes` lanes only, two handles take the same fused calls, one with the labels' overlay and one without, alternated
window by window (median of `--repeats`), then their compose kernel times (profile_kernels) in alternating rounds.  The
labels touch about 25.6 k of the canvas's 4.15 M pixels, so the difference is expected inside the run-to-run spread.

    python tools/bench_compose.py [--frames 16] [--lanes 16] [--window 2.0] [--repeats 3] [--labels]"""
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

from bench_nv12 import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--lanes", type=int, default=16)
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--labels", action="store_true", help="labels on against labels off (see above)")
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from bench import H, UI, W, make_clip

    if not torch.cuda.is_available():
        raise SystemExit("bench_compose.py needs an H100: the magnification core has no CPU fallback")
    before = card()
    lib = capi.lib()
    nv12_to_bgr, bgr_to_nv12 = lib.mc_debug_nv12_to_bgr, lib.mc_debug_bgr_to_nv12
    nv12_to_bgr.restype = bgr_to_nv12.restype = C.c_int
    cfg = L.ProcessorConfig(magnification=L.toParams(L.MagUiValues(
        L.MagnificationMode.Laplace, UI["amplification"], UI["wavelength"], UI["low"], UI["high"], UI["chroma"], UI["levels"],
        UI["fps"])))
    T, split = args.frames, capi.MC_SPLIT_LEFT_RIGHT
    cw, ch = L.MagnificationProcessor.compose_geometry(cfg, W, H, 3, split)
    assert (cw, ch) == (2 * W, H)
    lane_nv, canvas_nv = W * H * 3 // 2, cw * ch * 3 // 2

    def nv12(f):
        i420, n = cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420).ravel(), W * H
        uv = np.stack([i420[n:n + n // 4], i420[n + n // 4:]], -1).reshape(H // 2, W)
        return np.concatenate([i420[:n].reshape(H, W), uv])

    if args.labels:
        return labels_main(args, cfg, nv12, cw, ch, lane_nv, canvas_nv, before)
    results = {}
    for lanes in (1, args.lanes):
        v = T * lanes
        clip = make_clip(2, lanes)   # [2][lanes][H][W][3]: two distinct frame sets, repeated over the clip
        nv = np.stack([np.stack([nv12(f) for f in fs]) for fs in clip])
        d_nv = torch.from_numpy(nv[np.arange(v) // lanes % 2, np.arange(v) % lanes]).cuda()   # [v][3H/2][W]
        planes_in = capi.McNv12(d_nv.data_ptr(), d_nv.data_ptr() + W * H, W, lane_nv)
        d_canvas = torch.empty((v, canvas_nv), dtype=torch.uint8, device="cuda")
        canvas = capi.McCanvas(capi.MC_CANVAS_NV12, d_canvas.data_ptr(), d_canvas.data_ptr() + cw * ch, cw, canvas_nv)
        planes_out = capi.McNv12(d_canvas.data_ptr(), d_canvas.data_ptr() + cw * ch, cw, canvas_nv)
        d_out = torch.empty((v, H, W, 3), dtype=torch.uint8, device="cuda")
        d_orig = torch.empty((v, H, W, 3), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        fused_ch, sep_ch = L.ProcessingChainB200(0, lanes=lanes), L.ProcessingChainB200(0, lanes=lanes)

        def fused(k):
            flags, _ = fused_ch.magnifier.chain_compose_nv12_device(planes_in, T, W, H, cfg, split, canvas)
            fused_ch.magnifier.sync()

        def separate(k):
            sep_ch.process_nv12_device(planes_in, T, W, H, cfg, d_out.data_ptr(), 3 * W)
            sep_ch.magnifier.sync()
            assert nv12_to_bgr(C.byref(planes_in), W, H, v, C.c_void_p(d_orig.data_ptr()), C.c_size_t(3 * W)) == 0
            bgr = torch.cat([d_orig, d_out], dim=2)   # [v][H][2W][3]
            assert bgr_to_nv12(C.c_void_p(bgr.data_ptr()), C.c_size_t(3 * cw), cw, ch, v, None, C.byref(planes_out)) == 0
            torch.cuda.synchronize()

        paths = {"fused": fused, "separate": separate}
        for fn in paths.values():   # warm-up: module load, scratch allocation, the lanes' first frames
            fn(0)
            fn(1)
        rates = {k: [] for k in paths}
        for _ in range(args.repeats):
            for k, fn in paths.items():
                n, dt = timed(fn, args.window)
                rates[k].append(n * v / dt)
        fps = {k: statistics.median(r) for k, r in rates.items()}

        m = fused_ch.magnifier
        m.set_option("profile_kernels", 1)
        m.profile_read()
        n_prof = 10
        for i in range(n_prof):
            m.chain_compose_nv12_device(planes_in, T, W, H, cfg, split, canvas)
        prof = m.profile_read()
        m.set_option("profile_kernels", 0)
        launches, total_ms = prof[("compose", 0)]
        assert launches == n_prof
        compose_s = total_ms * 1e-3 / launches
        nbytes = (1.5 * W * H + 3 * W * H + 1.5 * cw * ch) * v
        results[f"lanes_{lanes}"] = {
            "virtual_lanes": v,
            "frames_per_s": {k: round(r, 1) for k, r in fps.items()},
            "fused_over_separate": round(fps["fused"] / fps["separate"], 3),
            "compose_us_per_launch": round(compose_s * 1e6, 2),
            "compose_us_per_canvas": round(compose_s * 1e6 / v, 3),
            "compose_bytes_per_canvas": nbytes / v,
            "compose_TBps": round(nbytes / compose_s / 1e12, 3),
            "compose_share_of_3.35TBps": round(nbytes / compose_s / 3.35e12, 3),
        }
        for chn in (fused_ch, sep_ch):
            chn.magnifier.close()
        del d_nv, d_canvas, d_out, d_orig
        torch.cuda.empty_cache()
    after = card()
    result = {
        "workload": f"Laplace {W}x{H} NV12 in, {UI['levels']} levels, LeftRight into a {cw}x{ch} NV12 canvas, clips of {T}",
        **results, "window_s": args.window, "repeats": args.repeats, "card_before": before, "card_after": after,
    }
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')})", flush=True)
    print(json.dumps(result), flush=True)


def labels_main(args, cfg, nv12, cw, ch, lane_nv, canvas_nv, before):
    import numpy as np
    import torch
    import lvm_b200 as L
    from lvm_b200 import capi
    from lvm_b200.labels import export_labels
    from bench import H, UI, W, make_clip

    T, lanes, split = args.frames, args.lanes, capi.MC_SPLIT_LEFT_RIGHT
    v = T * lanes
    ov = export_labels(cw, ch, split)
    clip = make_clip(2, lanes)
    nv = np.stack([np.stack([nv12(f) for f in fs]) for fs in clip])
    d_nv = torch.from_numpy(nv[np.arange(v) // lanes % 2, np.arange(v) % lanes]).cuda()
    planes_in = capi.McNv12(d_nv.data_ptr(), d_nv.data_ptr() + W * H, W, lane_nv)
    chains, canvases = {}, {}
    for k in ("labels", "plain"):
        d = torch.empty((v, canvas_nv), dtype=torch.uint8, device="cuda")
        canvases[k] = (d, capi.McCanvas(capi.MC_CANVAS_NV12, d.data_ptr(), d.data_ptr() + cw * ch, cw, canvas_nv))
        chains[k] = L.ProcessingChainB200(0, lanes=lanes)
    chains["labels"].magnifier.set_overlay(ov)

    def call(k):
        return lambda i: (chains[k].magnifier.chain_compose_nv12_device(planes_in, T, W, H, cfg, split, canvases[k][1]),
                          chains[k].magnifier.sync())

    paths = {k: call(k) for k in chains}
    for fn in paths.values():
        fn(0)
        fn(1)
    # the two handles ran the same frames: their canvases differ only inside the labels' rects
    diff = (canvases["labels"][0] != canvases["plain"][0]).reshape(v, -1)[:, :cw * ch].reshape(v, ch, cw)
    outside = diff.clone()
    for x, y, w, h in ov.boxes():
        outside[:, y:y + h, x:x + w] = False
    assert not bool(outside.any()) and bool(diff.any())
    rates = {k: [] for k in paths}
    for _ in range(args.repeats):
        for k, fn in paths.items():
            n, dt = timed(fn, args.window)
            rates[k].append(n * v / dt)
    kernel_us = {k: [] for k in paths}
    n_prof = 10
    for _ in range(args.repeats):
        for k in paths:
            m = chains[k].magnifier
            m.set_option("profile_kernels", 1)
            m.profile_read()
            for _i in range(n_prof):
                m.chain_compose_nv12_device(planes_in, T, W, H, cfg, split, canvases[k][1])
            launches, total_ms = m.profile_read()[("compose", 0)]
            m.set_option("profile_kernels", 0)
            assert launches == n_prof
            kernel_us[k].append(total_ms * 1e3 / launches)
    result = {
        "workload": f"Laplace {W}x{H} NV12 in, {UI['levels']} levels, {lanes} lanes, LeftRight into a {cw}x{ch} NV12 canvas, "
                    f"clips of {T}, labels on / off",
        "virtual_lanes": v,
        "label_rects": ov.boxes(), "label_pixels": sum(w * h for *_, w, h in ov.boxes()), "label_maps": len(ov.palette),
        "frames_per_s": {k: [round(r, 1) for r in rs] for k, rs in rates.items()},
        "frames_per_s_median": {k: round(statistics.median(rs), 1) for k, rs in rates.items()},
        "compose_us_per_launch": {k: [round(t, 2) for t in ts] for k, ts in kernel_us.items()},
        "compose_us_per_launch_median": {k: round(statistics.median(ts), 2) for k, ts in kernel_us.items()},
        "window_s": args.window, "repeats": args.repeats, "card_before": before, "card_after": card(),
    }
    print(f"card: {before.get('name')}, power limit {before.get('power.limit')}, SM clock {before.get('clocks.sm')} "
          f"(max {before.get('clocks.max.sm')})", flush=True)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
