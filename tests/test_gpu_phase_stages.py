"""Phase (Riesz) mode stage by stage, through the read-only taps "oct", "amp", "t_c", "t_s", "amplified" and "collapsed"
(mc_get_state) and the 13 state planes.

Every stage is teacher-forced: its reference is computed on the host from the device's own previous tap (or from the
state planes read before the frame call), so each comparison isolates one kernel:

  k_lab16           oct[0] == the lab16 tap's L * f32(100 / 16384), and == L of cv2.cvtColor(u8 / 255, BGR2Lab): bit for bit
  k_riesz_analysis  old.lowpass[i] == filter2D(oct[i], HP), oct[i+1] == filter2D(oct[i], 2 LP)[::2, ::2] (cv2, REFLECT_101):
                    bit for bit
  k_riesz_phase     the Riesz pair == filter2D(band, [-.2 -.48 0 .48 .2]) and its transpose, and amp: bit for bit.  The
                    new phases, the 8 DF-II registers, t_c and t_s equal, pixel by pixel, an f32 mirror of the kernel (every
                    op a correctly rounded one, the filter coefficients applied in float64) evaluated with
                    phi = acos(tmp) + k ulp for one k, |k| <= 2: CUDA's accuracy table bounds acosf by 2 ulp.  The clamp
                    branch (|tmp| > 1 -> +-1 rad) and the NaN patch (xy_sq == 0) take no k.
  k_riesz_amplify   an f32 mirror (the symmetric 13-tap pairs of g13 with fmaf, correctly rounded divide and sqrt,
                    THRESH_TRUNC) with cos / sin of the truncated magnitude off by (kc, ks) ulp, |k| <= 2 (sincosf's
                    bound), equal pixel by pixel with equal NaN masks.  Against the reference's own ops (GaussianBlur +
                    sepFilter2D + divide, libm cosf / sinf) within AMP_REF_TOL of the level's largest band or pair
                    magnitude times 1 + thresh: the two blurs sum in different orders (g13 is bit-equal to sepFilter2D
                    on about two thirds of the samples), which moves the magnitude m2 <= thresh by a few f32 ulp of
                    itself, and sincosf is not libm.
  k_riesz_collapse  cv2.add(filter2D(injectZerosEven(resize_NEAREST(collapsed[i+1] or oct[levels-1])), 2 LP),
                    filter2D(amplified[i], HP)): bit for bit, NaN positions included.  filter2D leaves out the zero
                    corner taps of HP, so a NaN of the amplified band (its blurred amplitude is 0 where L is 0) reaches
                    77 outputs, not 81.
  k_riesz_egress    the float output tap vs cv2.cvtColor(merge(collapsed[0], a, b of the lab16 tap), Lab2BGR): <= 8e-6
                    (the inverse's match to cv2; 7.7e-6 on saturated frames on an H100), NaN L' included (cv2 gives
                    1.0); a NaN L' gives exactly the egress's white, 1 - 2^-24 in every channel, as a clipped linear 1.0
                    does; the u8 output == convertTo of the float tap, byte for byte.

The clamp branch of the phase kernel is reached only where xy_sq == 0: with correctly rounded ops sqrt(fl(q_real^2) +
xy_sq) >= |q_real| unless q_real^2 underflows, and a subnormal q_real^2 plus a non-zero xy_sq (at least 2^-149) exceeds
q_real^2.  There the direction qx / xy_sqrt is infinite or NaN, so only the clamp's sign reaches the phase: a clamp to
+-pi instead of +-1 rad gives the same state, and no test can tell them apart.

The API's level clamp (both sides of a level that is halved exceed 5 pixels) keeps the Riesz residual at 6 pixels or more
a side and the smallest band level at 11 or more.  Lanes that did not run in a frame call (first frame, held) are not
compared with the mirrors: their taps keep what an earlier frame left, which is asserted."""
import collections
import math

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs, u8_diff
import np_model as M
from test_gpu_color_stages import fma32

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64

STATE = ("old.lowpass", "old.rx", "old.ry", "phase.c", "phase.s", "lo.r0.c", "lo.r0.s", "lo.r1.c", "lo.r1.s",
         "hi.r0.c", "hi.r0.s", "hi.r1.c", "hi.r1.s")
TAPS = ("oct", "amp", "t_c", "t_s", "amplified", "collapsed")
HP, LP2, RZ = O.HIGHPASS_9x9, (O.LOWPASS_9x9 * F32(2.0)).astype(F32), O.RIESZ_TAPS
ULP_K = (-2, -1, 0, 1, 2)
AMP_REF_TOL = 2.0 ** -19   # 1.05 * 2^-20 measured on an H100 80GB HBM3 (700 W), 0.28 * 2^-20 on the CPU emulation
# the egress's white: a linear value clipped to 1 (or NaN) through fmaf(1.055, 1, -0.055), 1 - 2^-24
WHITE = fma32(F32(1.055), 1.0, F32(-0.055))


def eff_levels(w, h, levels):
    return min(max(levels, 1), O.calculate_max_levels(w, h))


def f2d(img, k):
    return O._filter2d(np.ascontiguousarray(img, F32), k)


def same(a, b):
    """element-wise equality with NaN == NaN"""
    return (a == b) | (np.isnan(a) & np.isnan(b))


def ulp_shift(x, k):
    """x moved k f32 ulp (towards +inf for k > 0)"""
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf if k > 0 else -np.inf)).astype(F32)
    return x


class Handle:
    """A Phase handle fed [lanes][h][w][3] u8 frames, with its taps and state planes as [lanes][rows][cols]."""

    def __init__(self, lanes=1, options=()):
        self.p = L.MagnificationProcessor(0, lanes=lanes)
        self.p.set_option("keep_float_output", 1)
        for k, v in options:
            self.p.set_option(k, v)
        self.lanes = lanes

    def frame(self, frames, cfg):
        lanes, h, w, c = frames.shape
        buf = np.ascontiguousarray(frames)
        out = np.zeros_like(buf)
        produced = self.p.process_host(buf.ctypes.data, w, h, c, w * c, cfg, out.ctypes.data, w * c)
        return produced, out

    def tap(self, name, level=0):
        a = self.p.get_state(name, level)
        return None if a is None else a[:, 0]

    def states(self, levels):
        return {(n, i): self.tap(n, i) for n in STATE for i in range(levels - 1)}

    def taps(self, levels):
        return {(n, i): self.tap(n, i) for n in TAPS for i in range(levels)}

    def close(self):
        self.p.close()


# ---- host references ---------------------------------------------------------------------------------------------------
def muld(x, s):
    """cv::multiply(Mat, double): f32(double(x) * s)"""
    return (x.astype(F64) * F64(s)).astype(F32)


def iir_step(ph, r0, r1, b, a):
    """iir_step (DF-II) on f32 planes; b = (b0, b1, b2), a = (1, a1, a2) as double"""
    y = muld(ph, b[0]) + r0
    return y, (muld(ph, b[1]) + r1) - muld(y, a[1]), muld(ph, b[2]) - muld(y, a[2])


def phase_mirror(low, rx, ry, plow, prx, pry, st, flo, fhi):
    """k_riesz_phase's per-pixel arithmetic on f32 planes.  st: the 10 phase / register planes before the frame.
    -> (amp, branch masks, {k: outputs with phi = acos + k ulp})"""
    with np.errstate(all="ignore"):
        q_real = (low * plow + rx * prx) + ry * pry
        neg = -low
        qx = prx * neg + rx * plow
        qy = pry * neg + ry * plow
        xy_sq = qx * qx + qy * qy
        q_amp = np.sqrt(q_real * q_real + xy_sq)
        tmp = q_real / q_amp
        amp = np.sqrt(q_amp)
        xy_sqrt = np.sqrt(xy_sq)
        ox, oy = qx / xy_sqrt, qy / xy_sqrt
        acos = np.arccos(np.clip(tmp.astype(F64), -1.0, 1.0)).astype(F32)
        clamp = (tmp < -1) | (tmp > 1)
        out = {}
        for k in ULP_K:
            phi = np.where(tmp < -1, F32(-1), np.where(tmp > 1, F32(1), ulp_shift(acos, k))).astype(F32)
            pd_c, pd_s = ox * phi, oy * phi
            pd_c = np.where(np.isnan(pd_c), F32(0), pd_c)
            pd_s = np.where(np.isnan(pd_s), F32(0), pd_s)
            r = {"phase.c": st["phase.c"] + pd_c, "phase.s": st["phase.s"] + pd_s}
            y = {}
            for f, (b, a) in (("lo", flo), ("hi", fhi)):
                for cs in "cs":
                    y[f, cs], r[f"{f}.r0.{cs}"], r[f"{f}.r1.{cs}"] = iir_step(r[f"phase.{cs}"], st[f"{f}.r0.{cs}"],
                                                                             st[f"{f}.r1.{cs}"], b, a)
            r["t_c"] = (y["hi", "c"] - y["lo", "c"]) * amp
            r["t_s"] = (y["hi", "s"] - y["lo", "s"]) * amp
            out[k] = r
    return amp, {"clamp": clamp, "nan_patch": xy_sq == 0}, out


def g13_taps():
    """gaussian_kernel_13_3: cv::getGaussianKernel(13, 3, CV_32F), normalised in double and narrowed"""
    t = [math.exp(-0.5 / 9.0 * (i - 6.0) * (i - 6.0)) for i in range(13)]
    s = 0.0
    for v in t:
        s += v
    return [F32(v * (1.0 / s)) for v in t]


def g13_blur(p):
    """k_riesz_amplify's separable blur of one f32 plane: rows then columns, acc = k6 v6, then fmaf(k[6+j],
    v[6-j] + v[6+j], acc) for j = 1..6, reflect-101 borders"""
    g = g13_taps()

    def rows(q):
        n = q.shape[1]
        pad = q[:, M.reflect101(np.arange(-6, n + 6), n)]
        acc = (g[6] * pad[:, 6:6 + n]).astype(F32)
        for j in range(1, 7):
            acc = fma32(pad[:, 6 - j:6 - j + n] + pad[:, 6 + j:6 + j + n], g[6 + j], acc)
        return acc
    return rows(rows(p.astype(F32)).T).T


def amplify_mirror(amp, tc, ts, low, rx, ry, alpha, thresh):
    """-> (candidates [25][h][w], masks): out for every (kc, ks) ulp offset of cos / sin"""
    b0, b1, b2 = g13_blur(amp), g13_blur(tc), g13_blur(ts)
    with np.errstate(all="ignore"):
        c, s = b1 / b0, b2 / b0
        mag = np.sqrt(c * c + s * s)
        m2 = mag * F32(alpha)
        trunc = m2 > F32(thresh)
        m2 = np.where(trunc, F32(thresh), m2).astype(F32)
        pair = (rx * c + ry * s) / mag
        pair = np.where(np.isnan(pair), F32(0), pair)
        pc, ps = np.cos(m2.astype(F64)).astype(F32), np.sin(m2.astype(F64)).astype(F32)
        cands = np.stack([low * ulp_shift(pc, kc) - pair * ulp_shift(ps, ks) for kc in ULP_K for ks in ULP_K])
    return cands, {"trunc": trunc, "amp_nan": b0 == 0}


def amplify_reference(amp, tc, ts, low, rx, ry, alpha, thresh):
    """The blur and divide of RieszLevel::normalize and amplify() with the reference's own ops (cv2, libm cosf / sinf),
    from the phase kernel's amp and (hiIIR - loIIR) * amp"""
    kern = cv2.getGaussianKernel(13, 3.0, cv2.CV_32F)
    blurred = cv2.GaussianBlur(amp, (13, 13), 3.0)
    with np.errstate(all="ignore"):
        c, s = (cv2.divide(cv2.sepFilter2D(t, -1, kern, kern, anchor=(-1, -1), delta=0,
                                           borderType=cv2.BORDER_REFLECT_101), blurred) for t in (tc, ts))
        mag = cv2.sqrt(cv2.add(cv2.multiply(c, c), cv2.multiply(s, s)))
        _, m2 = cv2.threshold(O._scale(mag, alpha), float(thresh), 0, cv2.THRESH_TRUNC)
        pc, ps = O.cos_sin(m2)
        pair = O._patch_nans(cv2.divide(cv2.add(cv2.multiply(rx, c), cv2.multiply(ry, s)), mag))
        return cv2.subtract(cv2.multiply(low, pc), cv2.multiply(pair, ps))


def collapse_reference(coarse, amplified):
    h, w = amplified.shape
    up = cv2.resize(np.ascontiguousarray(coarse), (w, h), interpolation=cv2.INTER_NEAREST)
    upz = np.zeros_like(up)
    upz[::2, ::2] = up[::2, ::2]
    return cv2.add(f2d(upz, LP2), f2d(amplified, HP))


# ---- the stage checker (shared with tests/test_emu_phase_stages.py) -------------------------------------------------------
def check_frame(hd, frames, out, ops, before, prev, lv, prm, rebuild, stats):
    """Every stage of the frame call that just returned `out`.  ops[k] in {"run", "first", "hold"}; before: the 13 state
    planes read before the call (None on a fresh handle); prev: the taps read before the call; rebuild: the cutoffs
    changed (the prior is this frame's own band and pair, the registers start at zero)."""
    lanes, h, w, _ = frames.shape
    run = [k for k in range(lanes) if ops[k] == "run"]
    lab = hd.p.get_state("lab16", 0)
    octs = [hd.tap("oct", i) for i in range(lv)]
    assert hd.tap("oct", lv) is None and hd.tap("amp", lv - 1) is None and hd.tap("collapsed", lv - 1) is None
    after = hd.states(lv)
    for k in range(lanes):
        if ops[k] == "hold":
            for key, v in before.items():
                assert np.array_equal(after[key][k], v[k]), (key, k)
            for i in range(lv):
                assert np.array_equal(octs[i][k], prev["oct", i][k]), i
            continue
        # k_lab16
        L0 = cv2.cvtColor(O._u8_to_f32_scaled(frames[k], 1.0 / 255.0), cv2.COLOR_BGR2Lab)[..., 0]
        assert np.array_equal(octs[0][k], (lab[k, 0] * F32(100.0 / 16384.0)).astype(F32)), k
        assert np.array_equal(octs[0][k], L0), k
        # k_riesz_analysis
        for i in range(lv - 1):
            o = octs[i][k]
            assert np.array_equal(after["old.lowpass", i][k], f2d(o, HP)), (k, i)
            assert np.array_equal(octs[i + 1][k], f2d(o, LP2)[::2, ::2]), (k, i)
        if ops[k] == "first":
            for i in range(lv - 1):
                for n in STATE[1:]:
                    assert not after[n, i][k].any(), (k, i, n)
    # the phase kernel's taps exist when it ran on some lane; lanes that did not run keep the earlier contents
    assert (hd.tap("amp", 0) is not None) == bool(run)
    synth = bool(run) and not prm.get("analysis_only")
    assert (hd.tap("amplified", 0) is not None) == synth and (hd.tap("collapsed", 0) is not None) == synth
    for nm in TAPS[1:]:
        for i in range(lv - 1):
            cur, old = hd.tap(nm, i), prev[nm, i]
            if cur is not None and old is not None:
                for k in range(lanes):
                    if ops[k] != "run":
                        assert np.array_equal(cur[k], old[k], equal_nan=True), (nm, i, k)
    fps = prm["fps"]
    flo = (L.butterworth(2, prm["lo"] / (fps / 2.0))[1], L.butterworth(2, prm["lo"] / (fps / 2.0))[0])
    fhi = (L.butterworth(2, prm["hi"] / (fps / 2.0))[1], L.butterworth(2, prm["hi"] / (fps / 2.0))[0])
    thresh = F32(prm["coWavelength"] * (math.pi / 100.0))   # the UI's wavelength w gives coWavelength 100 - w
    fout = hd.p.float_output(w, h, 3) if synth else None
    for k in run:
        amplified = {}
        for i in range(lv - 1):
            band = after["old.lowpass", i][k]
            rx, ry = after["old.rx", i][k], after["old.ry", i][k]
            assert np.array_equal(rx, f2d(band, RZ)), (k, i)
            assert np.array_equal(ry, f2d(band, RZ.T.copy())), (k, i)
            if rebuild:
                prior = (band, rx, ry)
                st = {n: np.zeros_like(band) for n in STATE[3:]}
            else:
                prior = tuple(before[n, i][k] for n in STATE[:3])
                st = {n: before[n, i][k] for n in STATE[3:]}
            amp, masks, cand = phase_mirror(band, rx, ry, *prior, st, flo, fhi)
            got = {n: after[n, i][k] for n in STATE[3:]}
            got["t_c"], got["t_s"] = hd.tap("t_c", i)[k], hd.tap("t_s", i)[k]
            assert np.array_equal(hd.tap("amp", i)[k], amp, equal_nan=True), (k, i)
            ok = np.zeros(band.shape, bool)
            for kk in ULP_K:
                ok |= np.logical_and.reduce([same(got[n], cand[kk][n]) for n in got])
            assert ok.all(), (k, i, int((~ok).sum()), np.argwhere(~ok)[:4].tolist())
            stats["clamp"] += int(masks["clamp"].sum())
            assert not (masks["clamp"] & ~masks["nan_patch"]).any()   # see the module docstring
            stats["nan_patch"] += int(masks["nan_patch"].sum())
            if not synth:
                continue
            # k_riesz_amplify, from the phase kernel's taps
            tc, ts = got["t_c"], got["t_s"]
            amplified[i] = hd.tap("amplified", i)[k]
            cands, am = amplify_mirror(amp, tc, ts, band, rx, ry, prm["alpha"], thresh)
            okm = np.logical_or.reduce([same(amplified[i], c) for c in cands])
            assert okm.all(), (k, i, int((~okm).sum()), np.argwhere(~okm)[:4].tolist())
            stats["trunc"] += int(am["trunc"].sum())
            stats["no_trunc"] += int((~am["trunc"] & ~np.isnan(cands[12])).sum())
            stats["amp_nan"] += int(am["amp_nan"].sum())
            if thresh == 0:   # cos 0 = 1, sin 0 = 0: the band itself, NaN where the blurred amplitude is 0
                fin = ~am["amp_nan"]
                assert np.array_equal(amplified[i][fin], band[fin]) and np.isnan(amplified[i][~fin]).all()
            ref = amplify_reference(amp, tc, ts, band, rx, ry, prm["alpha"], thresh)
            assert np.array_equal(np.isnan(ref), np.isnan(amplified[i])), (k, i)
            # the blurs' relative difference moves the magnitude m2 <= thresh by that much of itself
            scale = max(float(np.abs(band).max()), float(np.abs(rx).max()), float(np.abs(ry).max()), 1e-30) * (1 + thresh)
            fin = ~np.isnan(ref)
            err = float(np.abs(amplified[i][fin] - ref[fin]).max()) if fin.any() else 0.0
            stats["amp_ref_err"] = max(stats["amp_ref_err"], err / scale)
            assert err <= AMP_REF_TOL * scale, (k, i, err / scale)
        if not synth:
            continue
        # k_riesz_collapse, level by level from the device's own coarser result
        collapsed = [hd.tap("collapsed", i)[k] for i in range(lv - 1)]
        for i in range(lv - 2, -1, -1):
            coarse = collapsed[i + 1] if i + 1 < lv - 1 else octs[lv - 1][k]
            ref = collapse_reference(coarse, amplified[i])
            assert np.array_equal(collapsed[i], ref, equal_nan=True), \
                (k, i, int((~same(collapsed[i], ref)).sum()), np.argwhere(~same(collapsed[i], ref))[:4].tolist())
        stats["nan_L"] += int(np.isnan(collapsed[0]).sum())
        # k_riesz_egress
        A = (lab[k, 1] * F32(1.0 / 64.0) - F32(128.0)).astype(F32)
        B = (lab[k, 2] * F32(1.0 / 64.0) - F32(128.0)).astype(F32)
        ref = cv2.cvtColor(cv2.merge([collapsed[0], A, B]), cv2.COLOR_Lab2BGR)
        if prm.get("egress_cv2", True):
            assert float(np.abs(fout[k] - ref).max()) <= 8e-6, k           # cv2 makes a NaN L' white: 1.0
        assert (fout[k][np.isnan(collapsed[0])] == WHITE).all(), k
        assert np.array_equal(out[k], O._f32_to_u8(fout[k], 255.0, 1.0 / 255.0)), k


# ---- content -------------------------------------------------------------------------------------------------------------
def content(kind, t, lanes, w, h, rng):
    """[lanes][h][w][3] u8 frame t: synth_frame, a black rectangle in it, a windowboxed picture (black all round),
    impulses on grey, or saturated black / white with a 1 LSB dither"""
    f = np.stack([synth_frame(t, w, h, 3, seed=70 * k) for k in range(lanes)])
    if kind == "blackrect":                      # 192 x 128: rows 40-80, columns 60-120
        f[:, h * 5 // 16:h * 10 // 16, w * 5 // 16:w * 10 // 16] = 0
    elif kind == "windowbox":
        bh, bw = max(h // 8, 5), max(w // 8, 5)
        f[:, :bh], f[:, -bh:], f[:, :, :bw], f[:, :, -bw:] = 0, 0, 0, 0
    elif kind == "impulses":
        g = np.full(f.shape, 60, np.int32) + rng.integers(0, 2, size=f.shape)
        g.reshape(lanes, h * w, 3)[:, rng.integers(0, h * w, size=max(1, h * w // 50))] = 250
        f = g.astype(np.uint8)
    elif kind == "saturated":
        g = np.where(f > 128, 255, 0) + rng.integers(-1, 2, size=f.shape)
        f = np.clip(g, 0, 255).astype(np.uint8)
    return np.ascontiguousarray(f)


def frame_launches(lv, ops, analysis_only=False):
    """lab16 + an analysis per band level; + phase, amplify and collapse per band level and the egress"""
    nb = lv - 1
    if all(o == "first" for o in ops):
        return 1 + nb
    if "run" not in ops or analysis_only:
        return 1 + 2 * nb
    return 2 + 4 * nb


def run_phase(w, h, lanes=1, levels=8, n=3, kind="synth", alpha=50, wavelength=50.0, lo=0.4, hi=3.0, fps=30.0,
              options=(), events=None, oracle=False, seed=0):
    """n frame calls through a handle, every one checked stage by stage; with `oracle` (1 lane) also free-running
    against the oracle at <= 3 LSB.  events[t]: [("restart", k) | ("hold", k, on) | ("cutoffs", lo, hi)] before
    frame t.  -> branch counters"""
    rng = np.random.default_rng(seed)
    lv = eff_levels(w, h, levels)
    assert lv >= 2
    hd = Handle(lanes, options)
    op = O.MagnificationProcessor() if oracle else None
    stats = collections.Counter()
    stats["amp_ref_err"] = 0.0
    first, held = [True] * lanes, [False] * lanes
    analysis_only = dict(options).get("analysis_only", 0) == 1
    for t in range(n):
        rebuild = False
        for e in (events or {}).get(t, []):
            if e[0] == "restart":
                hd.p.restart_lane(e[1])
                first[e[1]] = True
            elif e[0] == "hold":
                hd.p.hold_lane(e[1], e[2])
                held[e[1]] = bool(e[2])
            else:
                rebuild = (lo, hi) != e[1:]
                lo, hi = e[1:]
        ops = ["hold" if held[k] else "first" if first[k] else "run" for k in range(lanes)]
        rebuild = rebuild and "run" in ops
        cfg, ocfg = make_cfgs(O.MODE_PHASE, alpha, wavelength, lo, hi, 0, levels, fps)
        before = hd.states(lv) if t > 0 else None
        prev = hd.taps(lv)
        frames = content(kind, t, lanes, w, h, rng)
        n0 = hd.p.launch_count
        produced, out = hd.frame(frames, cfg)
        assert hd.p.launch_count - n0 == frame_launches(lv, ops, analysis_only), (t, ops)
        assert bool(produced) == ("run" in ops and not analysis_only), t
        prm = dict(alpha=alpha, coWavelength=ocfg.magnification.coWavelength, lo=lo, hi=hi, fps=fps, analysis_only=analysis_only)
        check_frame(hd, frames, out, ops, before, prev, lv, prm, rebuild, stats)
        if op is not None:
            oprod, oout = op.process(frames[0], ocfg)
            assert bool(oprod) == bool(produced)
            if produced:
                assert int(u8_diff(out[0], oout).max()) <= 3, (t, int(u8_diff(out[0], oout).max()))
        for k in range(lanes):
            first[k] = first[k] and held[k]
    hd.close()
    return stats


# ---- the seam sweep ------------------------------------------------------------------------------------------------------
# Around the 64 x 16 tiles of the 9x9 kernels (interior when 4 pixels of halo fit: w >= 132, h >= 36 for a second tile)
# and of amplify (8 / 6 pixels of halo: w >= 136, h >= 38), the 32 x 16 tile of the phase kernel, every width residue
# mod 8 at level 0 (filter2D's scalar tail columns x >= w & ~7) and more residues deeper, odd heights, and the smallest
# sizes the clamp allows (11 x 11: one band level of 11 x 11 over a residual of 6 x 6).
SWEEP = [(11, 11), (12, 13), (13, 21), (31, 17), (32, 16), (33, 15), (63, 33), (64, 31), (65, 32), (66, 37),
         (67, 36), (68, 38), (70, 39), (96, 48), (131, 36), (132, 37), (135, 40), (136, 35), (139, 51), (197, 71)]
SWEEP_CASES = [(w, h, (1, 3)[i % 2], i // 2 % 2) for i, (w, h) in enumerate(SWEEP)]


@pytest.mark.parametrize("w,h,lanes,tma", SWEEP_CASES)
def test_every_stage_on_the_seam_sweep(w, h, lanes, tma):
    assert {x % 8 for x, _ in SWEEP} == set(range(8))
    run_phase(w, h, lanes, n=3, options=(("use_tma", tma),), seed=w * 1000 + h)


KINDS = ("blackrect", "windowbox", "impulses", "saturated")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("tma", [0, 1])
def test_every_stage_on_flat_black_impulse_and_saturated_content(kind, tma):
    """192 x 128, the deepest pyramid (5 levels): the NaN of a black area (blurred amplitude 0) runs through amplify,
    the collapse and the egress, and the phase kernel takes its NaN patch (xy_sq == 0).  Its clamp branch needs
    q_real^2 to underflow: |tmp| > 1 cannot happen otherwise with correctly rounded ops.  The faint edge of a deep
    level's filter support next to black borders reaches that (values of 1e-20 and less)."""
    black = kind in ("blackrect", "windowbox")
    s = run_phase(192, 128, 1, levels=8, n=3, kind=kind, options=(("use_tma", tma),), oracle=black)
    if black:
        assert s["nan_patch"] > 0 and s["amp_nan"] > 0 and s["nan_L"] > 0, s
    if kind == "windowbox":
        assert s["clamp"] > 0, s


@pytest.mark.parametrize("alpha,wavelength,truncates", [(150, 80.0, True), (2, 0.0, False), (50, 100.0, True)])
def test_amplify_with_and_without_truncation(alpha, wavelength, truncates):
    """thresh = coWavelength * pi / 100 with coWavelength = 100 - the UI's wavelength: a high amplification truncates
    on some pixels, a low one on none; coWavelength 0 makes thresh 0, where the amplified band is the band itself"""
    s = run_phase(139, 51, 3, levels=4, n=4, kind="blackrect", alpha=alpha, wavelength=wavelength)
    assert (s["trunc"] > 0) == truncates and (s["no_trunc"] > 0) == (wavelength != 100.0), s


def test_blackrect_end_to_end_regression():
    """The black rectangle: the collapse reaches 77 outputs from a NaN of the amplified band, as filter2D does — the
    4 diagonal pixels beyond are the picture, not white; u8 within 3 LSB of the oracle over 6 frames"""
    s = run_phase(192, 128, 1, levels=4, n=6, kind="blackrect", oracle=True)
    assert s["nan_L"] > 0


def test_blackrect_clip_equals_frame_calls():
    cfg = make_cfgs(O.MODE_PHASE, 50, 50.0, 0.4, 3.0, 0, 4, 30.0)[0]
    w, h, lanes = 192, 128, 2
    rng = np.random.default_rng(0)
    frames = np.stack([content("blackrect", t, lanes, w, h, rng) for t in range(5)])
    a, b = L.MagnificationProcessor(0, lanes=lanes), L.MagnificationProcessor(0, lanes=lanes)
    flags, outc = a.process_clip(frames, cfg)
    assert flags[1:].all()
    for t in range(5):
        prod, o = b.process_image(frames[t], cfg)
        assert bool(prod) == bool(flags[t].any())
        if prod:
            assert np.array_equal(outc[t], o), t
    assert all(a.state_dims(nm, 0) == (0, 0, 0) for nm in TAPS)   # a clip call: no taps
    a.close()
    b.close()


# ---- lifecycle -----------------------------------------------------------------------------------------------------------
def test_lanes_run_restart_and_hold():
    """3 lanes: lane 1 restarted at frame 3 (FIRST while the others run), lane 2 held over frames 3-5 (its 13 state
    planes and its taps unchanged), at frame 5 a frame of FIRST + HOLD only (the phase kernel runs on no lane), then all
    run"""
    events = {3: [("restart", 1), ("hold", 2, 1)], 5: [("hold", 0, 1), ("restart", 1)],
              6: [("hold", 0, 0), ("hold", 2, 0)]}
    run_phase(135, 40, 3, levels=4, n=8, kind="blackrect", events=events)


def test_cutoff_change_rebuilds_the_prior_from_zeroed_registers():
    events = {3: [("cutoffs", 0.8, 3.0)], 5: [("cutoffs", 0.8, 2.0)]}
    run_phase(131, 37, 1, levels=4, n=7, events=events)
    run_phase(70, 39, 3, levels=3, n=5, events={2: [("cutoffs", 0.5, 2.5)]}, kind="windowbox")


def test_analysis_only_has_no_synthesis_taps():
    run_phase(96, 48, 2, levels=3, n=4, options=(("analysis_only", 1),))


def test_taps_are_read_only_and_absent_without_a_frame():
    hd = Handle(2)
    cfg = make_cfgs(O.MODE_PHASE, 50, 50.0, 0.4, 3.0, 0, 3, 30.0)[0]
    rng = np.random.default_rng(1)
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in TAPS)
    hd.frame(content("synth", 0, 2, 40, 24, rng), cfg)             # all lanes first: the octaves only
    assert hd.tap("oct", 0) is not None and hd.tap("amp", 0) is None and hd.tap("amplified", 0) is None
    hd.frame(content("synth", 1, 2, 40, 24, rng), cfg)
    for nm in TAPS:
        a = hd.p.get_state(nm, 0)
        assert a is not None and a.shape == (2, 1, 24, 40)
        with pytest.raises(L.MagcoreError) as e:
            hd.p.set_state(nm, 0, a)
        assert e.value.status == capi.MC_ERR_INVALID
    assert hd.p.state_dims("oct", 2) == (6, 10, 1) and hd.p.state_dims("oct", 3) == (0, 0, 0)
    assert hd.p.state_dims("collapsed", 1) == (12, 20, 1) and hd.p.state_dims("collapsed", 2) == (0, 0, 0)
    hd.p.reset()
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in TAPS)
    hd.frame(content("synth", 0, 2, 40, 24, rng), cfg)
    hd.frame(content("synth", 1, 2, 40, 24, rng), cfg)
    hd.frame(content("synth", 2, 2, 40, 24, rng)[..., :1].copy(), cfg)   # gray input passes through
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in TAPS)
    hd.frame(content("synth", 3, 2, 48, 24, rng), cfg)             # new geometry: a first frame
    assert hd.tap("oct", 0) is not None and hd.tap("amp", 0) is None
    hd.frame(content("synth", 4, 2, 48, 24, rng), make_cfgs(O.MODE_LAPLACE, 50, 50.0, 0.4, 3.0, 0, 3, 30.0)[0])
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in TAPS)
    hd.close()
