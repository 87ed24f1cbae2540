#!/usr/bin/env python
"""Randomised parity hunt: random frame sizes, contents (noise, flats, gradients, saturation, letterbox, impulses),
modes, levels and parameters — with mid-stream parameter changes and resets — through the CUDA path and the checker
(the reference's compiled code, oracle/_ref, else the oracle).  Prints every case that breaks the tolerances.

    MC_EMU=1 python tests/tools/fuzz_parity.py --cases 200 --seed 0      # on the CUDA-on-CPU emulation (no GPU)
    python tests/tools/fuzz_parity.py --cases 500                         # on an H100
    MC_EMU=1 python tests/tools/fuzz_parity.py --chain --cases 500        # the fused front of the chain (ROI / INTER_AREA /
                                                                    # gray): original tap bit-exact, frame <= 1 LSB
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def make_frames(rng, w, h, c, n, kind):
    shape = (h, w, c) if c == 3 else (h, w)
    base = rng.integers(0, 256, size=shape).astype(np.float64)
    yy, xx = np.mgrid[0:h, 0:w]
    frames = []
    for t in range(n):
        if kind == "noise":
            f = base + rng.integers(-6, 7, size=shape)
        elif kind == "smooth":
            g = 128 + 90 * np.sin(xx / 9.0 + 0.4 * t) * np.cos(yy / 7.0)
            f = (g[..., None] + np.array([0, 15, -20])) if c == 3 else g
            f = f + rng.integers(-2, 3, size=shape)
        elif kind == "flat":
            f = np.full(shape, float(rng.integers(0, 256)))
        elif kind == "letterbox":
            f = base + rng.integers(-4, 5, size=shape)
            f[: h // 4] = 0
            f[h - h // 5:] = 0
        elif kind == "saturated":
            f = np.where(base > 128, 255.0, 0.0) + rng.integers(-1, 2, size=shape)
        elif kind == "impulses":
            f = np.full(shape, 20.0)
            idx = rng.integers(0, h * w, size=max(1, h * w // 50))
            f.reshape(h * w, -1)[idx] = 250
            f = f + rng.integers(0, 2, size=shape) * (t % 2)
        else:  # gradient
            g = xx * 255.0 / max(1, w - 1) + 3 * t
            f = (g[..., None] * np.array([1.0, 0.5, 0.25])) if c == 3 else g
        frames.append(np.clip(np.rint(f), 0, 255).astype(np.uint8))
    return frames


def fuzz_chain(args):
    import lvm_b200 as L
    from oracle import livim_oracle as O, livim_ref
    from common import make_cfgs
    R = livim_ref.load()
    assert R is not None, "the chain fuzz checks against the compiled reference (oracle/_ref)"
    rng = np.random.default_rng(args.seed)
    bad, t0 = 0, time.time()
    for case in range(args.cases):
        w, h, c = int(rng.integers(8, args.max_size + 40)), int(rng.integers(8, args.max_size + 40)), int(rng.choice([1, 3]))
        down, gray, roi_on = int(rng.choice([1, 2, 3, 4, 5, 7, 8, 0, 9])), bool(rng.random() < 0.4), bool(rng.random() < 0.6)
        roi = rng.uniform(-0.1, 1.1, size=4) if rng.random() < 0.3 else \
            (rng.uniform(0, 0.6), rng.uniform(0, 0.6), rng.uniform(0.05, 1.0), rng.uniform(0.05, 1.0))
        roi = [float(np.float32(v)) for v in roi]
        mode = int(rng.choice([O.MODE_LAPLACE, O.MODE_LAPLACE, O.MODE_PHASE, O.MODE_COLOR, O.MODE_NONE]))
        ui = {O.MODE_PHASE: (50, 50.0, 0.4, 3.0, 0), O.MODE_COLOR: (100, 0.0, 0.8, 1.2, 0)}.get(mode, (20, 50.0, 0.4, 3.0, 20))
        cfg, ocfg = make_cfgs(mode, *ui, int(rng.integers(1, 5)), 8.0)
        cfg.grayscale = ocfg.grayscale = gray
        cfg.preprocess, ocfg.preprocess = L.PreprocessParams(down, roi_on, *roi), O.PreprocessParams(down, roi_on, *roi)
        rcfg = livim_ref.to_ref_config(R, ocfg)
        chain, rchain = L.ProcessingChainB200(0), R.Chain()
        desc = f"chain case {case} seed {args.seed}: mode {mode} {w}x{h}x{c} down={down} gray={gray} roi_on={roi_on} roi={roi}"
        try:
            base = rng.integers(0, 256, size=(h, w, 3) if c == 3 else (h, w))
            for t in range(4):
                f = np.clip(base + rng.integers(-5, 6, size=base.shape), 0, 255).astype(np.uint8)
                cur, orig = chain.run_chain_once(L.Frame(image=f, seq=t), cfg)
                rcur, rorig, _, _, _ = rchain.process(f, rcfg)
                if orig.image.shape != rorig.shape or not np.array_equal(orig.image, rorig):
                    print("ORIGINAL TAP DIFFERS", desc, "frame", t)
                    bad += 1
                    break
                lim = 3 if mode == O.MODE_PHASE else 1
                if cur.image.shape != rcur.shape or int(np.abs(cur.image.astype(np.int32) - rcur.astype(np.int32)).max()) > lim:
                    print("FRAME DIFFERS", desc, "frame", t)
                    bad += 1
                    break
        except Exception as e:   # noqa: BLE001
            print("EXCEPTION", desc, repr(e)[:200])
            bad += 1
    print(f"{args.cases} chain cases, {bad} outside tolerance, {time.time() - t0:.0f} s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-size", type=int, default=120)
    ap.add_argument("--chain", action="store_true")
    ap.add_argument("--options", action="store_true", help="also switch random A/B kernel options on (Laplace)")
    args = ap.parse_args()
    if os.environ.get("MC_EMU") == "1":
        import conftest
        conftest.use_emulated_library(asan=os.environ.get("MC_EMU_ASAN") == "1")
    if args.chain:
        return fuzz_chain(args)
    import lvm_b200 as L
    from oracle import livim_oracle as O, livim_ref
    from common import make_cfgs
    R = livim_ref.load()
    rng = np.random.default_rng(args.seed)
    kinds = ["noise", "smooth", "flat", "letterbox", "saturated", "impulses", "gradient"]
    bad, t0 = 0, time.time()
    for case in range(args.cases):
        mode = int(rng.choice([O.MODE_LAPLACE, O.MODE_PHASE, O.MODE_COLOR]))
        w, h = int(rng.integers(6, args.max_size + 1)), int(rng.integers(6, args.max_size + 1))
        c = 3 if mode == O.MODE_PHASE or rng.random() < 0.7 else 1
        kind = str(rng.choice(kinds))
        if mode == O.MODE_COLOR and kind == "flat" and not os.environ.get("FUZZ_KEEP_COLOR_FLAT"):
            # a temporally constant window is degenerate in the reference itself: its temporal DFT is exactly zero for
            # some window lengths and rounding noise for others (OpenCV's per-length FFT kernels), and the min-max
            # normalisation stretches that noise to full range — not reproducible by any other FFT (DESIGN.md §2)
            kind = "noise"
        n = int(rng.integers(3, 8)) if mode != O.MODE_COLOR else int(rng.integers(4, 22))
        fps = float(rng.choice([8.0, 12.0, 30.0]))

        def params():
            lo = float(rng.choice([0.0, 0.4, 0.8, 2.0]))
            return (int(rng.choice([0, 5, 20, 50, 150])), float(rng.choice([0.0, 10.0, 50.0, 90.0, 100.0])), lo,
                    lo + float(rng.choice([0.0, 0.4, 2.5, 20.0])), int(rng.choice([0, 30, 100])), int(rng.integers(1, 9)))
        ui = params()
        if mode == O.MODE_PHASE and ui[3] > fps / 2:
            # beyond Nyquist the reference's Butterworth design has poles outside the unit circle (the UI clamps to Nyquist):
            # the registers explode within a few frames and any rounding difference with them
            ui = ui[:3] + (fps / 2,) + ui[4:]
        frames = make_frames(rng, w, h, c, n, kind)
        cfg, ocfg = make_cfgs(mode, *ui, fps)
        proc = L.MagnificationProcessor(0)
        opts = []
        if args.options:
            opts = [k for k in ("prefetch_state", "ingest_warps", "band_from_state", "faithful_level0", "use_tma")
                    if rng.random() < 0.4]
            for k in opts:
                proc.set_option(k, {"faithful_level0": 1, "ingest_warps": 4}.get(k, 0))
        if R is not None:
            ref, rcfg = R.Processor(), livim_ref.to_ref_config(R, ocfg)
        else:
            ref, rcfg = O.MagnificationProcessor(), ocfg
        change_at = int(rng.integers(2, n)) if rng.random() < 0.4 else -1
        reset_at = int(rng.integers(2, n)) if rng.random() < 0.15 else -1
        desc = (f"case {case} seed {args.seed}: mode {mode} {w}x{h}x{c} {kind} n={n} fps={fps} ui={ui} change@{change_at} "
                f"reset@{reset_at} options={opts}")
        if os.environ.get("FUZZ_VERBOSE"):
            print(desc, flush=True)
        try:
            for t, f in enumerate(frames):
                if t == change_at:   # non-structural change: same levels, new alpha / cutoffs / wavelength / chroma
                    u2 = params()
                    ui2 = (u2[0], u2[1], u2[2], min(u2[3], fps / 2) if mode == O.MODE_PHASE else u2[3], u2[4], ui[5])
                    desc += f" ui2={ui2}"
                    cfg, ocfg = make_cfgs(mode, *ui2, fps)
                    rcfg = livim_ref.to_ref_config(R, ocfg) if R is not None else ocfg
                if t == reset_at:
                    proc.reset()
                    ref.reset()
                produced, out = proc.process_image(f, cfg)
                rprod, rout = ref.process(f, rcfg)
                if produced != bool(rprod):
                    print("PRODUCED MISMATCH", desc, "frame", t, produced, rprod)
                    bad += 1
                    break
                if produced:
                    d = np.abs(out.astype(np.int32) - rout.astype(np.int32))
                    same = float((d == 0).mean())
                    lim = 3 if mode == O.MODE_PHASE else 1
                    if int(d.max()) > lim or same < (0.995 if mode == O.MODE_PHASE else 0.99):
                        print("DIFF", desc, "frame", t, "max", int(d.max()), "identical", round(same, 5))
                        bad += 1
                        break
        except Exception as e:   # noqa: BLE001
            print("EXCEPTION", desc, repr(e)[:200])
            bad += 1
        proc.close()
    print(f"{args.cases} cases, {bad} outside tolerance, {time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()
