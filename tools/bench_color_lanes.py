#!/usr/bin/env python
"""Color mode on a multi-lane handle whose lanes have their own windows (option "color_lane_lifecycle"): 1080p, 3 levels,
0.8-1.2 Hz at 30 fps (window 64), `lanes` device-resident streams (mc_process_device), timed with CUDA events.

  (a) steady state, every lane's window full: this build against --lib (for example the parent commit's build), the
      two alternated round by round in one process, and the last step's outputs of both compared byte for byte;
  (b) staggered joins: from a fresh handle lane k is restarted at frame 4k, so the lanes warm up at different lengths;
  (c) steady state with one lane held.

Each scenario also reports launches per step (mc_launch_count) and, from a separate run with profile_kernels, cuFFT
executions per step; the card's name and power limit are read in the same call.

    python tools/bench_color_lanes.py [--lanes 16] [--steps 120] [--rounds 3] [--lib path/to/parent/libmagcore_b200.so]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_clip import card  # noqa: E402

W, H, CH, LEVELS, FPS, WINDOW = 1920, 1080, 3, 3, 30.0, 64
T = 8   # distinct frames per lane, cycled


def load(lib_path):
    """-> (MagnificationProcessor class bound to that library, McParams of the workload)"""
    from lvm_b200 import capi
    capi.LIB_PATH, capi._lib = os.path.abspath(lib_path), None
    lib = capi.lib()
    import lvm_b200 as L
    p = capi.McParams()
    lib.mc_params_from_ui(C.byref(p), capi.MODE_COLOR, 100, 0.0, 0.8, 1.2, 0, LEVELS, FPS)
    return L.MagnificationProcessor, lib, p


class Arm:
    """One library's handle over the shared device frames."""

    def __init__(self, lib_path, lanes, clip, lifecycle):
        import torch
        self.cls, self.lib, self.p = load(lib_path)
        self.lanes, self.clip, self.lifecycle = lanes, clip, lifecycle
        self.out = torch.full((lanes, H, W, CH), 0, dtype=torch.uint8, device="cuda")
        self.proc = None
        self.i = 0

    def fresh(self, profile=False):
        from lvm_b200 import capi
        if self.proc:
            self.proc.close()
        capi._lib = self.lib   # a processor binds the library current at its creation
        self.proc = self.cls(0, lanes=self.lanes)
        if self.lifecycle:
            self.proc.set_option("color_lane_lifecycle", 1)
        if profile:
            self.proc.set_option("profile_kernels", 1)
        self.i = 0

    def step(self, events=()):
        for kind, k in events:
            self.proc.restart_lane(k) if kind == "restart" else self.proc.hold_lane(k, 1)
        row = W * CH
        assert self.proc.process_device(self.clip[self.i % T].data_ptr(), W, H, CH, row, self.p, self.out.data_ptr(), row) is not None
        self.i += 1


def timed(arm, steps, events_at=lambda i: ()):
    """-> (frames/s over `steps` steps, launches per step)"""
    import torch
    stream = torch.cuda.ExternalStream(arm.proc.stream)
    l0 = arm.proc.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        arm.step(events_at(arm.i))
    e1.record(stream)
    torch.cuda.synchronize()
    return arm.lanes * steps / (e0.elapsed_time(e1) * 1e-3), (arm.proc.launch_count - l0) / steps


def staggered(lanes):
    return lambda i: [("restart", i // 4)] if i % 4 == 0 and 0 < i // 4 < lanes else []


def cufft_per_step(arm, warm, steps, events_at):
    """profile_kernels run: cuFFT executions (R2C + C2R) per step over `steps` steps after `warm` steps"""
    import torch
    arm.fresh(profile=True)
    for _ in range(warm):
        arm.step(events_at(arm.i))
    torch.cuda.synchronize()
    arm.proc.profile_read()
    for _ in range(steps):
        arm.step(events_at(arm.i))
    prof = arm.proc.profile_read()
    return sum(prof.get((k, 0), (0, 0.0))[0] for k in ("cufft_r2c", "cufft_c2r")) / steps


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=16)
    ap.add_argument("--steps", type=int, default=120)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--lib", default=None, help="also time this libmagcore_b200.so in (a), alternated with the in-tree build")
    args = ap.parse_args()
    import torch
    from bench import make_clip
    lanes = args.lanes
    clip = torch.from_numpy(make_clip(T, lanes)).cuda()
    here = os.path.join(ROOT, "live-video-magnification_b200", "libmagcore_b200.so")
    res = {"workload": f"{lanes} x {W}x{H}x{CH}, Color, {LEVELS} levels, 0.8-1.2 Hz at {FPS:g} fps (window {WINDOW}), "
                       f"device frames", "card": card()}

    # (a) steady state, alternated with --lib
    arms = {"this": Arm(here, lanes, clip, True)}
    if args.lib:
        arms["lib"] = Arm(args.lib, lanes, clip, False)
    fps = {k: [] for k in arms}
    launches = {}
    for a in arms.values():
        a.fresh()
        for _ in range(WINDOW + 8):
            a.step()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, a in arms.items():
            f, n = timed(a, args.steps)
            fps[k].append(f)
            launches[k] = n
    a_res = {k: {"fps_per_round": fps[k], "fps_median": median(fps[k]), "launches_per_step": launches[k]} for k in arms}
    if args.lib:
        # both handles saw the same frames in the same order: their last outputs are compared byte for byte
        a_res["outputs_equal_lib"] = bool(torch.equal(arms["this"].out, arms["lib"].out))
        a_res["lanes_produced_equal_lib"] = bool(np.array_equal(arms["this"].proc.lane_produced(), arms["lib"].proc.lane_produced()))
    a_res["cufft_execs_per_step"] = cufft_per_step(arms["this"], WINDOW + 8, 8, lambda i: ())
    res["a_steady"] = a_res

    this = arms["this"]
    # (b) staggered joins: lane k restarted at frame 4k; timed over the first 4 * lanes + WINDOW frames
    n_b = 4 * lanes + WINDOW
    fb = []
    for _ in range(args.rounds):
        this.fresh()
        f, n = timed(this, n_b, staggered(lanes))
        fb.append(f)
    res["b_staggered"] = {"frames": n_b, "fps_per_round": fb, "fps_median": median(fb), "launches_per_step": n,
                          "cufft_execs_per_step": cufft_per_step(this, 0, n_b, staggered(lanes))}

    # (c) one lane held in the steady state
    fc = []
    this.fresh()
    for _ in range(WINDOW + 8):
        this.step()
    this.proc.hold_lane(lanes // 2, 1)
    for _ in range(args.rounds):
        f, n = timed(this, args.steps)
        fc.append(f)
    res["c_one_held"] = {"fps_per_round": fc, "fps_median": median(fc), "launches_per_step": n}
    this.proc.hold_lane(lanes // 2, 0)
    for a in arms.values():
        a.proc.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
