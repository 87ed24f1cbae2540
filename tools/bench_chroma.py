#!/usr/bin/env python
"""bench.py's workload (`lanes` 1080p streams, Motion (Laplace), 6 levels) at a chosen chroma attenuation, and the
interface bytes of the synthesis kernels counted from shapes.

At chroma 0 the library synthesises the L planes only (DESIGN.md §4: L-only synthesis), while bench.py's kernel_table
counts every channel for the egress and the collapses, so at chroma 0 it overstates their bytes.  This script prints
both counts (band_from_state on, the library default), then times device-resident steps (mc_process_device on `lanes`
lanes, CUDA events over --steps steps, --rounds rounds, after a warm-up) at --chroma, with the card's name and power
limit.  --lib times another build's library on the same workload (for example the parent commit's build).

    python tools/bench_chroma.py [--chroma 30] [--lanes 64] [--steps 300] [--rounds 3] [--lib path/to/libmagcore_b200.so]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CH, H, LEVELS, UI, W, kernel_table, level_pixels, make_clip  # noqa: E402
from tools.bench_clip import card  # noqa: E402


def counted_bytes(lanes):
    """-> {"full": {kernel: bytes}, "luma": {...}} per step.  L-only synthesis reads one plane of hi_1 / lo_1, of cur_2
    and of the collapses' sources instead of three; the Lab16 input read and the u8 write are unchanged."""
    p = level_pixels(W, H, LEVELS)
    prof = {("ingest_lab", 0): (1, 1.0), ("egress", 0): (1, 1.0)}
    prof.update({("level", l): (1, 1.0) for l in range(1, LEVELS)})
    prof.update({("collapse", l): (1, 1.0) for l in range(2, LEVELS - 1)})
    full = {t["kernel"]: t["interface_bytes"] for t in kernel_table(prof, lanes, band_from_state=True)}
    luma = dict(full)
    luma["egress[0]"] = (3 * CH * p[0] + 8 * p[1] + (8 if LEVELS == 3 else 4) * p[2]) * lanes
    for l in range(2, LEVELS - 1):
        luma[f"collapse[{l}]"] = full[f"collapse[{l}]"] // CH
    return {"full": full, "luma": luma}


def time_steps(args):
    import torch
    from lvm_b200 import capi
    if args.lib:
        capi.LIB_PATH, capi._lib = os.path.abspath(args.lib), None
    import lvm_b200 as L

    p = capi.McParams()
    capi.lib().mc_params_from_ui(C.byref(p), capi.MODE_LAPLACE, UI["amplification"], UI["wavelength"], UI["low"], UI["high"],
                                 args.chroma, UI["levels"], UI["fps"])
    lanes, T, row = args.lanes, 8, W * CH
    clip = torch.from_numpy(make_clip(T, lanes)).cuda()
    out = torch.empty((lanes, H, W, CH), dtype=torch.uint8, device="cuda")
    proc = L.MagnificationProcessor(0, lanes=lanes)
    stream = torch.cuda.ExternalStream(proc.stream)
    i = 0

    def step():
        nonlocal i
        assert proc.process_device(clip[i % T].data_ptr(), W, H, CH, row, p, out.data_ptr(), row)
        i += 1

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    fps = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        e1.record(stream)
        torch.cuda.synchronize()
        fps.append(lanes * args.steps / (e0.elapsed_time(e1) * 1e-3))
    proc.close()
    return fps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chroma", type=int, default=30, help="UI chroma attenuation (percent)")
    ap.add_argument("--lanes", type=int, default=64)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--lib", default=None, help="time this libmagcore_b200.so instead of the in-tree build")
    ap.add_argument("--bytes-only", action="store_true", help="print the counted bytes and stop (no GPU needed)")
    args = ap.parse_args()
    res = {"workload": f"{args.lanes} x 1920x1080x3, Laplace, {LEVELS} levels, chroma {args.chroma}",
           "counted_bytes_per_step": counted_bytes(args.lanes)}
    if not args.bytes_only:
        res.update({"lib": args.lib or "in-tree", "fps_per_round": time_steps(args), "card": card()})
        res["fps_median"] = sorted(res["fps_per_round"])[len(res["fps_per_round"]) // 2]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
