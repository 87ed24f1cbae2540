#!/usr/bin/env python
"""Torch-free GPU probe (seconds, for tight GPU-time budgets): parity of the Laplace path against the checker on a
small and a 1080p clip, then the per-kernel device-time table (profile_kernels) of the 1080p bench workload through
the blocking host API.  Prints one JSON line.

    python tests/tools/quick_gpu_probe.py                 # parity + one table (PROBE_LANES, default 8)
    python tests/tools/quick_gpu_probe.py --ab 8,32       # A/B of the kernel options at those lane counts:
                                                    # the option sets in PROBE_VARIANTS (JSON list), default: ingest_warps 2 / 4, prefetch_state 0, band_from_state 0
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    t00 = time.time()
    import lvm_b200 as L
    from lvm_b200.synth import synth_frame
    from oracle import livim_oracle as O, livim_ref
    from common import make_cfgs
    out = {}
    pw, ph = int(os.environ.get("PROBE_W", "1920")), int(os.environ.get("PROBE_H", "1080"))
    R = livim_ref.load()
    for (w, h, levels, n) in (() if os.environ.get("PROBE_SKIP_PARITY") == "1" else ((320, 240, 4, 6), (pw, ph, 6, 3))):
        cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, levels)
        proc = L.MagnificationProcessor(0)
        ref = R.Processor() if R is not None else O.MagnificationProcessor()
        rcfg = livim_ref.to_ref_config(R, ocfg) if R is not None else ocfg
        worst, ndiff = 0, 0
        for t in range(n):
            f = synth_frame(t, w, h, 3)
            _, o = proc.process_image(f, cfg)
            _, ro = ref.process(f, rcfg)
            d = np.abs(o.astype(np.int32) - ro.astype(np.int32))
            worst, ndiff = max(worst, int(d.max())), ndiff + int((d > 0).sum())
        out[f"parity_{w}x{h}"] = {"max_u8_diff": worst, "differing": ndiff, "checker": "reference" if R is not None else "oracle"}
        proc.close()
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 6)
    # PROBE_CLIP: what the frames look like.  "synthetic" = the bench clip (six gratings down to 8 px + noise: neighbouring
    # pixels often fall into different cells of the Lab LUT), "smooth" = a natural-video-like gradient field with +-1
    # noise, "noise" = white noise (worst case for the LUT gathers).  Comparing ingest_lab across them shows how much of
    # its time is L1 wavefronts of the exact-LUT gathers (the hypothesis behind a lane mapping with 32 adjacent pixels).
    kind = os.environ.get("PROBE_CLIP", "synthetic")
    if kind == "synthetic":
        base = [synth_frame(t, pw, ph, 3) for t in range(2)]
    else:
        rng = np.random.default_rng(0)
        yy, xx = np.mgrid[0:ph, 0:pw]
        base = []
        for t in range(2):
            if kind == "smooth":
                g = 128 + 60 * np.sin(xx / 180.0 + 0.1 * t) * np.cos(yy / 140.0)
                f = g[..., None] + np.array([0.0, 12.0, -18.0]) + rng.integers(-1, 2, size=(ph, pw, 3))
            else:
                f = rng.integers(0, 256, size=(ph, pw, 3)).astype(np.float64)
            base.append(np.clip(np.rint(f), 0, 255).astype(np.uint8))
    out["clip"] = kind

    def table_for(lanes, options):
        clip = [np.stack([np.roll(base[t], (11 * k, 37 * k), axis=(0, 1)) for k in range(lanes)]) for t in range(2)]
        if lanes == 1:
            clip = [c[0] for c in clip]          # a single stream takes plain HxWxC frames
        proc = L.MagnificationProcessor(0, lanes=lanes)
        for k, v in options.items():
            proc.set_option(k, v)
        for i in range(3):
            proc.process_image(clip[i % 2], cfg)
        proc.set_option("profile_kernels", 1)
        for i in range(8):
            proc.process_image(clip[i % 2], cfg)
        prof = proc.profile_read()
        proc.close()
        table = sorted(((f"{k}[{lvl}]", tms / n * 1e3) for (k, lvl), (n, tms) in prof.items()), key=lambda r: -r[1])
        step = sum(us for _, us in table)
        return {"lanes": lanes, "options": options, "kernels_us": {k: round(us, 1) for k, us in table},
                "step_us": round(step, 1), "fps_device_kernels_only": round(lanes / (step * 1e-6), 1)}

    if "--ab" in sys.argv:
        lane_list = [int(x) for x in sys.argv[sys.argv.index("--ab") + 1].split(",")]
        # every variant in its own process: a kernel fault poisons the CUDA context of the process it happens in
        import subprocess
        variants = json.loads(os.environ.get("PROBE_VARIANTS", "null")) or (
            {}, {"ingest_warps": 2}, {"ingest_warps": 4}, {"prefetch_state": 0}, {"band_from_state": 0},
            {"prefetch_state": 0, "band_from_state": 0})
        out["ab"] = []
        for n in lane_list:
            for o in variants:
                env = dict(os.environ, PROBE_LANES=str(n), PROBE_OPTIONS=json.dumps(o), PROBE_SKIP_PARITY="1")
                r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True, timeout=120)
                try:
                    out["ab"].append(json.loads(r.stdout.strip().splitlines()[-1]))
                except Exception:
                    out["ab"].append({"lanes": n, "options": o, "failed": (r.stderr or r.stdout)[-400:]})
    else:
        out.update(table_for(int(os.environ.get("PROBE_LANES", "8")), json.loads(os.environ.get("PROBE_OPTIONS", "{}"))))
    out["seconds"] = round(time.time() - t00, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
