#!/usr/bin/env python
"""One stream, one GPU: per-frame calls vs clips.

The workload is bench.py's (BASELINE.json configs[1]: Motion (Laplace) 1920x1080x3, 6 levels, IIR 0.4-3 Hz @30fps,
alpha=20) on ONE stream with the frames resident in HBM.  In one process, alternating in every round, it times
  - mc_process_device, one call per frame,
  - mc_process_clip_device with T = 8, 16, 32 frames per call,
  - for reference, mc_process_device on a T-lane handle (T independent streams per launch set, bench.py's lane batching),
with CUDA events on each handle's stream over windows of at least --seconds.  Every method walks the same 32-frame
sequence the same number of times, so the per-frame and clip outputs of the last pass are compared bit for bit.
A separate run with profile_kernels gives per-kernel times.  Reported: frames/s, the level kernels' counted bytes
(from shapes, SURVEY 8d) and roofline.frame = A_min(T) * fps / peak, with the card's name and power limit.

With --mode phase the workload is tools/mode_bench.py's `phase` config instead: Phase (Riesz) 1920x1080x3, 6 levels,
UI amplification 50, wavelength 50, 0.4-3 Hz @30fps, timed the same way.  Reported: frames/s, bit equality, per-kernel
times, the phase kernels' bytes per frame counted from shapes, and the clip scratch per frame.  A Phase handle's first
frame passes through, so only the handle's first frame is allowed not to produce.

    python tools/bench_clip.py [--mode laplace|phase] [--seconds 1.0] [--rounds 3] [--out result.json]
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import CH, H, LEVELS, UI, W, WORKLOAD, level_pixels, make_clip, measured_peaks  # noqa: E402

N = 32            # frames in the sequence every method walks (a multiple of every T)
TS = (8, 16, 32)


def counted_bytes(t_frames):
    """Level kernels' bytes per frame from shapes.  Frame kernel at level l: reads G_l and both states, writes both
    states and G_{l+1}: 16*C*P_l + 4*C*(P_l + P_{l+1}).  Clip kernel: reads G_l, writes G_{l+1} and the band M_l, and moves
    the two states once per clip: 4*C*P_l + 4*C*P_{l+1} + 4*C*P_l + 16*C*P_l / T."""
    p = level_pixels(W, H, LEVELS)
    frame = {l: 16 * CH * p[l] + 4 * CH * (p[l] + p[l + 1]) for l in range(1, LEVELS)}
    clip = {l: 8 * CH * p[l] + 4 * CH * p[l + 1] + 16 * CH * p[l] / t_frames for l in range(1, LEVELS)}
    return frame, clip


def a_min(t_frames):
    """SURVEY 8d with temporal batches of T: 2*C*P0 + 16*C*S/T, S = sum of P_1 .. P_{L-1}."""
    p = level_pixels(W, H, LEVELS)
    return 2 * CH * p[0] + 16 * CH * sum(p[1:LEVELS]) / t_frames


PHASE_UI = (50, 50.0, 0.4, 3.0, 0, LEVELS, 30.0)   # amplification, wavelength, low, high, chroma, levels, fps
PHASE_WORKLOAD = "Phase (Riesz) 1920x1080x3 BGR, 6 levels, UI amplification 50, wavelength 50, 0.4-3 Hz @30fps"


def riesz_levels(w, h, levels):
    """(w, h, pitch) of the Phase octaves 0 .. levels-1 (subsample(): ceil halving; rows padded to 32 floats)"""
    out = []
    for _ in range(levels):
        out.append((w, h, (w + 31) // 32 * 32))
        w, h = w // 2 + w % 2, h // 2 + h % 2
    return out


def phase_counted_bytes(t_frames):
    """The phase kernels' bytes per frame from shapes, per pitched band-level pixel (one L plane).  k_riesz_phase reads
    the band (4), the prior {low, Rx, Ry} (12) and the state (2 phases + 8 registers, 40) and writes Rx, Ry (8), the state
    (40) and amp, t_c, t_s (12): 116 B.  k_riesz_phase_clip moves per frame the band (4), Rx, Ry (8) and amp, t_c, t_s
    (12), and once per clip the prior and the state in (52) and out (52): 24 + 104 / T B."""
    px = sum(h * pitch for (_, h, pitch) in riesz_levels(W, H, LEVELS)[:LEVELS - 1])
    return px, 116 * px, (24 + 104 / t_frames) * px


def phase_clip_scratch_bytes():
    """Device scratch of a Phase clip per frame of one lane (RieszMode::Clip): every octave, the band and the Riesz
    pair of every band level, amp / t_c / t_s of the largest level, and the Lab int16 planes."""
    lv = riesz_levels(W, H, LEVELS)
    planes = [h * pitch for (_, h, pitch) in lv]
    floats = sum(planes) + 3 * sum(planes[:LEVELS - 1]) + 3 * planes[0]
    return 4 * floats + 2 * 3 * H * ((W + 63) // 64 * 64)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:   # the numbers are then reported without the card, and say so
        return {"name": None, "error": f"nvidia-smi: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="least length of one timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    ap.add_argument("--mode", choices=["laplace", "phase"], default="laplace")
    args = ap.parse_args()
    phase = args.mode == "phase"

    import torch
    import lvm_b200 as L
    from lvm_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py needs an H100: the magnification core has no CPU fallback")
    p = capi.McParams()
    if phase:
        capi.lib().mc_params_from_ui(C.byref(p), capi.MODE_PHASE, *PHASE_UI)
    else:
        capi.lib().mc_params_from_ui(C.byref(p), capi.MODE_LAPLACE, UI["amplification"], UI["wavelength"], UI["low"], UI["high"],
                                     UI["chroma"], UI["levels"], UI["fps"])
    row = W * CH
    frame_bytes = H * row
    d_in = torch.from_numpy(make_clip(N, 1)).cuda()                    # [N][1][H][W][3]
    base = d_in.data_ptr()

    class Method:
        def __init__(self, name, t_frames, lanes=1):
            self.name, self.t, self.lanes = name, t_frames, lanes
            self.proc = L.MagnificationProcessor(0, lanes=lanes)
            self.stream = torch.cuda.ExternalStream(self.proc.stream)
            self.out = torch.empty_like(d_in)
            self.fps = []
            self.fresh = phase   # Phase: the handle's first frame passes through

        def step(self):
            """the N-frame sequence once"""
            o = self.out.data_ptr()
            if self.name == "frame":
                for i in range(N):
                    assert self.proc.process_device(base + i * frame_bytes, W, H, CH, row, p, o + i * frame_bytes, row) or self.fresh
                    self.fresh = False
            elif self.name == "clip":
                for i in range(0, N, self.t):
                    f = self.proc.process_clip_device(base + i * frame_bytes, self.t, W, H, CH, row, p, o + i * frame_bytes, row)
                    assert f.all() or (self.fresh and f[1:].all())
                    self.fresh = False
            else:   # T lanes per launch set: N / T steps of T streams
                for i in range(0, N, self.lanes):
                    assert self.proc.process_device(base + i * frame_bytes, W, H, CH, row, p, o + i * frame_bytes, row) or self.fresh
                    self.fresh = False

        def time(self, steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.stream)
            for _ in range(steps):
                self.step()
            e1.record(self.stream)
            e1.synchronize()
            return e0.elapsed_time(e1) * 1e-3

    methods = [Method("frame", 1)] + [Method("clip", t) for t in TS] + [Method("lanes", 1, lanes=t) for t in TS]
    # warm-up of every shape, then the number of passes that makes the slowest window >= --seconds
    steps = 1
    for m in methods:
        m.step()
        torch.cuda.synchronize()
        steps = max(steps, math.ceil(args.seconds / m.time(1)))
    for _ in range(args.rounds):
        for m in methods:
            m.fps.append(steps * N / m.time(steps))
    torch.cuda.synchronize()

    ref = methods[0].out.cpu().numpy()
    equal = {f"T={m.t}": bool(np.array_equal(m.out.cpu().numpy(), ref)) for m in methods if m.name == "clip"}

    # per-kernel times: a separate run with event bracketing (profile_kernels), per frame of the stream
    kernels = {}
    for label, t_frames in (("frame", 1), ("clip T=16", 16)):
        pr = L.MagnificationProcessor(0)
        pr.set_option("profile_kernels", 1)
        o = torch.empty_like(d_in)
        for _ in range(2):
            for i in range(0, N, t_frames):
                if t_frames == 1:
                    pr.process_device(base + i * frame_bytes, W, H, CH, row, p, o.data_ptr() + i * frame_bytes, row)
                else:
                    pr.process_clip_device(base + i * frame_bytes, t_frames, W, H, CH, row, p, o.data_ptr() + i * frame_bytes, row)
            prof = pr.profile_read()   # the second pass is kept
        kernels[label] = {f"{k}[{lvl}]": round(ms * 1e3 / N, 2) for (k, lvl), (n, ms) in sorted(prof.items(), key=lambda x: -x[1][1])}
        pr.close()

    if phase:
        rates = {}
        for m in methods:
            key = "frame" if m.name == "frame" else f"{m.name} T={m.t if m.name == 'clip' else m.lanes}"
            rates[key] = {"fps": round(statistics.median(m.fps), 1), "fps_rounds": [round(x, 1) for x in m.fps]}
        px, frame_b, _ = phase_counted_bytes(1)
        result = {
            "workload": PHASE_WORKLOAD + ", one stream, frames in HBM",
            "card": card(),
            "unit": "frames/s (device-resident, CUDA events on the handle's stream, median of rounds)",
            "window_s_min": args.seconds, "passes_per_window": steps, "frames_per_pass": N,
            "rates": rates,
            "bit_equal_to_frame_calls": equal,
            "band_level_pixels": px,
            "counted_bytes_phase_kernels_MB_per_frame": {"frame_kernel": round(frame_b / 1e6, 1),
                                                         **{f"clip_kernel T={t}": round(phase_counted_bytes(t)[2] / 1e6, 1) for t in TS}},
            "clip_scratch_MB_per_frame": round(phase_clip_scratch_bytes() / 1e6, 1),
            "kernel_us_per_frame": kernels,
        }
        line = json.dumps(result)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                f.write(line + "\n")
        for m in methods:
            m.proc.close()
        if not all(equal.values()):
            raise SystemExit("clip outputs differ from per-frame outputs")
        return

    peak, peak_src = measured_peaks()
    frame_b, clip_b = counted_bytes(16)
    rates = {}
    for m in methods:
        fps = statistics.median(m.fps)
        key = "frame" if m.name == "frame" else f"{m.name} T={m.t if m.name == 'clip' else m.lanes}"
        t_eff = m.t if m.name == "clip" else 1
        rates[key] = {"fps": round(fps, 1), "fps_rounds": [round(x, 1) for x in m.fps],
                      "roofline_frame": round(a_min(t_eff) * fps / 1e9 / peak, 4) if m.name != "lanes" else None}
    result = {
        "workload": WORKLOAD + ", one stream, frames in HBM",
        "card": card(),
        "unit": "frames/s (device-resident, CUDA events on the handle's stream, median of rounds)",
        "window_s_min": args.seconds, "passes_per_window": steps, "frames_per_pass": N,
        "rates": rates,
        "bit_equal_to_frame_calls": equal,
        "counted_bytes_level1_T16": {"frame_kernel_MB": round(frame_b[1] / 1e6, 2), "clip_kernel_MB": round(clip_b[1] / 1e6, 2)},
        "counted_bytes_levels_T16": {"frame_kernel_MB": round(sum(frame_b.values()) / 1e6, 2),
                                     "clip_kernel_MB": round(sum(clip_b.values()) / 1e6, 2)},
        "a_min_MB": {f"T={t}": round(a_min(t) / 1e6, 2) for t in (1,) + TS},
        "peak_GBps": peak, "peak_source": peak_src,
        "kernel_us_per_frame": kernels,
    }
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for m in methods:
        m.proc.close()
    if not all(equal.values()):
        raise SystemExit("clip outputs differ from per-frame outputs")


if __name__ == "__main__":
    main()
