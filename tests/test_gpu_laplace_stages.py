"""Laplace (Motion) mode stage by stage, through the read-only tap "gauss" (the Gaussian pyramid G_1 .. G_levels of the
last frame call), "lab16", the state planes "lowpassHi" / "lowpassLo", "band" and the float output tap.

Every stage is teacher-forced: its reference is computed on the host from the device's own previous tap (or from state
set with mc_set_state), so each comparison isolates one kernel.  The band of a frame that runs is not visible directly:
a twin handle takes the same frame as its first frame, where hi = lo = the band (MagnifyCore.hpp:98-103).  The band
depends only on the frame, so the twin's "gauss" must equal the handle's bit for bit.

  k_ingest_lab    G_1 (3 channels, levels >= 2) == float64 pyrDown (reflect-101) of the decoded lab16 tap: a, b exactly
                  (multiples of 1/64 below 128 with weights summing to 256: every partial sum is representable), L within B
  k_down_strip    G_1 of gray frames (levels >= 2) vs float64 pyrDown of u8 * f32(1/255): within B; with faithful_level0
  / k_level l=0   level 0 is k_level<IN_LAB16 / IN_U8>, which also yields the level-0 band (within B')
  k_level         G_{l+1} vs float64 pyrDown of the device's G_l: within B.  The band (hi == lo after a first frame, bit
                  for bit) vs G_l - pyrUp64(G_{l+1}) with cv::pyrUp's border rule s[-1] := s[1], s[n] := s[n-1]: within B'.
                  The EMAs of a frame that runs: bit for bit against f32(DFMA(s, 1 - c, DMUL(x, c))), the form every
                  k_level and k_level_clip variant compiles `ema` to (one DMUL by c, one DFMA by 1 - c, F2F.F32.F64),
                  with the fused product evaluated exactly on the host (ema_exact).  The stored band
                  f32(f32(hi' - lo') * gain_l): bit for bit (+-0 on a first frame).
  k_collapse      "band" at levels 2 .. levels-2 == fma(pyrUp taps of cur_{l+1}, 1/64, m_l) with the pinned f32 taps
                  up3(a, b, c) = fma(b, 6, a) + c and up2(a, b) = (a + b) * 4, rows first: bit for bit
  egress          gray: the same mirror for cur_1 and the level-0 sums u, then fma(u, 1/64, u8 * f32(1/255)); float tap and
                  u8 bit for bit.  Colour: Lab' = (fma(u_L, 1/64, L), A + f32(u_A * chroma / 64), ...) exactly, and the
                  float tap within FLOAT_TWIN_TOL of cv2.cvtColor(Lab', Lab2BGR); u8 == convertTo of the float tap, and
                  within 1 LSB of convertTo of cv2's.

The bounds B and B'.  A pass of the pyrDown stencil c*6 + (b+d)*4 + a + e takes at most four f32 roundings (the * 4 is
exact; nvcc may fuse c*6 or (b+d)*4 into an FMA, which drops one), each at most 2^-24 of a partial sum bounded by the
pass's weighted absolute sum.  The row pass puts at most 4 * 2^-24 of that sum on each of its outputs; the column pass
weights them with the same kernel and adds its own four, and the * 1/256 is exact.  So |err| <= 8 * 2^-24 * S (+ higher
order terms) with S = pyrDown64(|x|), the float64 weighted absolute sum over the support, and B = 2^-20 * S is twice
that.  The band is G_l - pyrUp(G_{l+1}~), where G_{l+1}~ is the coarse window the tile computed itself: a tile next to
another may compute the shared coarse samples on its border path, whose contractions differ, so G_{l+1}~ is within
B_{l+1} of the tap.  pyrUp has four roundings over a kernel of weights summing to 1 and the subtraction one more, so
B' = 2^-20 * (|G_l| + pyrUp64(|G_{l+1}|) + pyrUp64(S_{l+1})) covers it.  Largest errors measured, in units of the bound:
see DESIGN.md §2 (SEEN holds them for a run).

A wrong neighbour, border source or tap is an error of one neighbour difference; check_sensitivity asserts that on the
seam content the neighbour differences exceed 2^10 B at most samples, so such a mistake is many bounds away."""
import collections
import ctypes as C
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.processor import _to_mc
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs
import np_model as M
from test_gpu_full_range import FLOAT_TWIN_TOL, content as full_range_content

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
EMU = os.environ.get("MC_EMU") == "1"
# largest |error| / bound over the checks run in this process (reported in DESIGN.md §2)
SEEN = collections.Counter()
UNIT = F32(0.003921568859368563)   # (float)(1/255)
INV64 = F32(1.0 / 64.0)


def eff_levels(w, h, levels):
    return min(max(levels, 1), O.calculate_max_levels(w, h))


# ---- exact f32 / f64 arithmetic on the host -----------------------------------------------------------------------------
def _round_to_odd(s, e):
    """s = RN64(x), e = x - s exactly: RO64(x) (the odd neighbour when x is not representable).  Rounding RO64(x) to
    f32 gives RN32(x): 53 >= 24 + 2 bits."""
    bits = s.view(np.int64)
    even = (bits & 1) == 0
    bump = (e != 0) & even
    return np.where(bump, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fma32(a, b, c):
    """fmaf(a, b, c) on f32 values, correctly rounded: a * b is exact in float64, the sum is rounded to odd there"""
    a, b, c = (np.asarray(v, F32).astype(F64) for v in (a, b, c))
    s, e = _two_sum(a * b, c)
    return _round_to_odd(np.asarray(s, F64), np.asarray(e, F64)).astype(F32)


def add32(a, b):
    return fma32(a, F32(1), b)


def mul32(a, b):
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)).astype(F32)


def ema_exact(s, x, omc, c):
    """f32(fma64(s, omc, x * c)): `ema` as k_level / k_level_clip compute it.  s * omc = A + B exactly (omc split into
    26 + 27 bits, s has 24); the three-term sum is evaluated in float64 and, where that can differ from the correctly
    rounded DFMA at the f32 rounding (within 8 float64 ulp of an f32 rounding midpoint), exactly with Fractions."""
    from fractions import Fraction
    s = np.asarray(s, F32).astype(F64)
    x = np.asarray(x, F32).astype(F64)
    p = x * F64(c)
    split = F64(134217729.0) * F64(omc)
    hi = split - (split - F64(omc))
    lo = F64(omc) - hi
    A, B = s * hi, s * lo
    t, e1 = _two_sum(A, p)
    d = t + (e1 + B)
    r = d.astype(F32)
    q = r.astype(F64)
    nb = np.nextafter(r, np.where(d > q, F32(np.inf), F32(-np.inf))).astype(F64)
    near = np.abs(d - (q + nb) / 2) <= 8 * np.spacing(np.abs(d))
    for i in zip(*np.nonzero(near)):
        ex = Fraction(float(A[i])) + Fraction(float(B[i])) + Fraction(float(p[i]))
        r[i] = F32(float(ex))   # Fraction -> float rounds correctly (the DFMA), then F2F.F32.F64
    return r


def unit_to_u8(f):
    """unit_to_u8 / cvt.rni.u8.f32 of fmaf(x, 255, 1/255): round half even, NaN and negatives 0, clamped to 255"""
    v = np.rint(fma32(f, F32(255), UNIT).astype(F64))
    return np.where(~(v > 0), 0, np.minimum(v, 255)).astype(np.uint8)


# ---- pyramid references ---------------------------------------------------------------------------------------------------
def pyr_down64(p):
    """float64 cv::pyrDown of [..., h, w] planes (reflect-101)"""
    p = np.asarray(p, F64)
    h, w = p.shape[-2:]
    xs = [M.reflect101(2 * np.arange((w + 1) // 2) + d, w) for d in (-2, -1, 0, 1, 2)]
    row = 6 * p[..., xs[2]] + 4 * (p[..., xs[1]] + p[..., xs[3]]) + p[..., xs[0]] + p[..., xs[4]]
    ys = [M.reflect101(2 * np.arange((h + 1) // 2) + d, h) for d in (-2, -1, 0, 1, 2)]
    return (6 * row[..., ys[2], :] + 4 * (row[..., ys[1], :] + row[..., ys[3], :]) + row[..., ys[0], :] + row[..., ys[4], :]) / 256


def _up_pass64(s, n_f):
    odd, im1, i0, ip1 = M._up_idx(n_f, s.shape[-1])
    return np.where(odd, 4 * (s[..., i0] + s[..., ip1]), s[..., im1] + 6 * s[..., i0] + s[..., ip1])


def pyr_up64(p, hw):
    """float64 cv::pyrUp of [..., hc, wc] to [..., h, w]: s[-1] := s[1], s[n] := s[n-1]"""
    r = _up_pass64(np.asarray(p, F64), hw[1])
    return np.swapaxes(_up_pass64(np.swapaxes(r, -1, -2), hw[0]), -1, -2) / 64


def _up_pass32(s, n_f):
    odd, im1, i0, ip1 = M._up_idx(n_f, s.shape[-1])
    up3 = add32(fma32(s[..., i0], F32(6), s[..., im1]), s[..., ip1])
    up2 = mul32(add32(s[..., i0], s[..., ip1]), F32(4))
    return np.where(odd, up2, up3).astype(F32)


def up_sum32(p, hw):
    """the synthesis kernels' pyrUp tap sums (before the exact 1/64) of f32 [..., hc, wc] at [..., h, w]: up3 / up2 rows
    first, then columns"""
    r = _up_pass32(np.asarray(p, F32), hw[1])
    return np.swapaxes(_up_pass32(np.swapaxes(r, -1, -2), hw[0]), -1, -2)


def check_bound(got, ref, bound, stats, key, ctx):
    err = np.abs(got.astype(F64) - ref)
    ratio = float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0
    stats[key] = max(stats[key], ratio)
    assert (err <= bound).all(), (ctx, key, ratio, np.argwhere(err > bound)[:4].tolist())


def check_sensitivity(src, bound, l, stats):
    """A wrong neighbour of the outermost tap moves an output by 1/256 of a neighbour difference of the input (the
    inner taps by more): the median of that, over the median bound, at pyramid step l"""
    d = np.abs(np.diff(np.asarray(src, F64), axis=-1)) / 256
    stats[f"sens{l}"] = float(np.median(d) / max(float(np.median(bound)), 1e-300))


# ---- the handle -----------------------------------------------------------------------------------------------------------
class Handle:
    """A Laplace handle fed [lanes][h][w][C] u8 frames; taps as [lanes][C][rows][cols]."""

    def __init__(self, lanes=1, options=()):
        self.p = L.MagnificationProcessor(0, lanes=lanes)
        self.p.set_option("keep_float_output", 1)
        self.options = dict(options)
        for k, v in options:
            self.p.set_option(k, v)
        self.lanes = lanes

    def frame(self, frames, params, pad=0, out=None):
        lanes, h, w, c = frames.shape
        step = w * c + pad
        buf = np.zeros((lanes, h, step), np.uint8)
        buf[:, :, : w * c] = frames.reshape(lanes, h, w * c)
        if out is None:
            out = np.full((lanes, h, step), 0xA5, np.uint8)
        produced = self.p.process_host(buf.ctypes.data, w, h, c, step, params, out.ctypes.data, step)
        return produced, out

    def tap(self, name, level=0):
        return self.p.get_state(name, level)

    def close(self):
        self.p.close()


def params(levels, alpha=20, wavelength=50.0, lo=0.4, hi=3.0, chroma=50, fps=30.0, co_low=None, co_high=None):
    p = _to_mc(make_cfgs(O.MODE_LAPLACE, alpha, wavelength, lo, hi, chroma, levels, fps)[0])
    if co_low is not None:
        p.coLow = co_low
    if co_high is not None:
        p.coHigh = co_high
    return p


def gains_of(p, lv, w, h):
    g = (C.c_float * (lv + 1))()
    q = capi.McParams.from_buffer_copy(p)
    q.levels = lv
    assert capi.lib().mc_motion_gains(C.byref(q), lv, w, h, g) == capi.MC_OK
    return [F32(v) for v in g]


def frame_launches(c, lv, ops, faithful, groups, motion):
    """ingest (+ nothing else for gray), one level kernel per level run, the faithful residual copy pair per run of
    first-frame lanes in each lane group, the collapses and the egress"""
    fused = c == 3 and not faithful and lv >= 2
    first_level = 1 if fused else (0 if (lv >= 2 or faithful) else lv)
    n = (1 if c == 3 else 0) * groups_n(groups) + (lv - first_level) * groups_n(groups)
    if faithful:
        for a, b in groups:
            runs, prev = 0, False
            for k in range(a, b):
                cur = ops[k] == "first"
                runs += cur and not prev
                prev = cur
            n += 2 * runs
    if motion:
        n += max(0, lv - 3) * groups_n(groups)
    return n + groups_n(groups)


def groups_n(groups):
    return len(groups)


def lane_groups(lanes, req):
    ng = req if req > 0 else min(2, lanes // 8)
    ng = max(1, min(ng, lanes))
    return [(lanes * g // ng, lanes * (g + 1) // ng) for g in range(ng)]


# ---- the stage checker (shared with tests/test_emu_laplace_stages.py) -----------------------------------------------------
def check_frame(hd, tw, frames, out, ops, prev, prm, stats, ctx):
    """Every stage of the frame call that just returned `out`.  ops[k] in {"run", "first", "hold"}; prev: the taps and
    state read before the call (after any mc_set_state); tw: the twin handle that took the same frame as a first frame."""
    lanes, h, w, c = frames.shape
    lv, faithful, from_state = prm["lv"], prm["faithful"], prm["from_state"]
    live = [k for k in range(lanes) if ops[k] != "hold"]
    motion = "run" in ops and lv >= 2
    G = {l: hd.tap("gauss", l) for l in range(1, lv + 1)}
    assert hd.p.state_dims("gauss", 0) == (0, 0, 0) and hd.p.state_dims("gauss", lv + 1) == (0, 0, 0)
    if lv == 1 and not faithful:
        assert G[1] is None
        return
    for l in G:
        assert G[l] is not None and G[l].shape == (lanes, c, (h + 2 ** l - 1) >> l, (w + 2 ** l - 1) >> l), (l, ctx)
    state_levels = [l for l in range(lv + 1) if hd.p.state_dims("lowpassHi", l)[0] > 0]
    hi = {l: hd.tap("lowpassHi", l) for l in state_levels}
    lo = {l: hd.tap("lowpassLo", l) for l in state_levels}
    band = {l: hd.tap("band", l) for l in range(lv + 1)}
    # held lanes: pyramid, state, band planes and output bytes untouched
    for k in range(lanes):
        if ops[k] != "hold":
            continue
        for name, d in (("gauss", G), ("hi", hi), ("lo", lo), ("band", band)):
            for l, v in d.items():
                if v is not None and prev[name].get(l) is not None:
                    assert np.array_equal(v[k], prev[name][l][k]), (ctx, name, l, k)
        assert (out[k] == 0xA5).all(), (ctx, k)
    # level 0 as the kernels read it
    if c == 3:
        lab = hd.tap("lab16", 0)
        G0 = np.stack([mul32(lab[:, 0], F32(100.0 / 16384.0)), fma32(lab[:, 1], INV64, F32(-128)),
                       fma32(lab[:, 2], INV64, F32(-128))], 1)
    else:
        G0 = mul32(np.moveaxis(frames, 3, 1).astype(F32), UNIT)
    Gd = {0: G0, **G}
    # the pyramid: G_{l+1} from the device's G_l
    for l in range(lv):
        src = Gd[l][live]
        ref = pyr_down64(src)
        bound = 2.0 ** -20 * pyr_down64(np.abs(src))
        got = Gd[l + 1][live]
        if l == 0 and c == 3 and not faithful:   # k_ingest_lab: a, b exact
            assert np.array_equal(got[:, 1:], ref[:, 1:].astype(F32)), ctx
            check_bound(got[:, :1], ref[:, :1], bound[:, :1], stats, "B", (ctx, "ingest L"))
        else:
            check_bound(got, ref, bound, stats, "B", (ctx, "down", l))
        if prm.get("sensitivity"):
            check_sensitivity(src, bound, l, stats)
    # the twin: same pyramid bit for bit; its hi == lo is this frame's band
    Gt = {l: tw.tap("gauss", l) for l in range(1, lv + 1)}
    for l in G:
        assert np.array_equal(Gt[l][live], G[l][live]), (ctx, "twin gauss", l)
    band_levels = [l for l in range(lv) if (l >= 1 or faithful)]
    bnd = {}
    for l in band_levels:
        th, tl = tw.tap("lowpassHi", l), tw.tap("lowpassLo", l)
        assert np.array_equal(th, tl), (ctx, "twin hi == lo", l)
        bnd[l] = th
        fine, coarse = Gd[l][live], Gd[l + 1][live]
        ref = fine.astype(F64) - pyr_up64(coarse, fine.shape[-2:])
        S = pyr_down64(np.abs(fine))
        bound = 2.0 ** -20 * (np.abs(fine) + pyr_up64(np.abs(coarse), fine.shape[-2:]) + pyr_up64(S, fine.shape[-2:]))
        check_bound(th[live], ref, bound, stats, "B'", (ctx, "band", l))
    if faithful:   # the residual of a first frame: hi = lo = G_levels
        for k in live:
            if ops[k] == "first":
                assert np.array_equal(hi[lv][k], G[lv][k]) and np.array_equal(lo[lv][k], G[lv][k]), (ctx, k)
    # the temporal filter, per lane
    c_hi, c_lo = prm["co_high"], prm["co_low"] if prm["co_low"] != 0 else 0.01
    gains = prm["gains"]
    m = {}
    for l in band_levels:
        nh, nl = hi[l].copy(), lo[l].copy()
        for k in live:
            if ops[k] == "first":
                assert np.array_equal(hi[l][k], bnd[l][k]) and np.array_equal(lo[l][k], bnd[l][k]), (ctx, l, k)
            else:
                eh = ema_exact(prev["hi"][l][k], bnd[l][k], 1 - c_hi, c_hi)
                el = ema_exact(prev["lo"][l][k], bnd[l][k], 1 - c_lo, c_lo)
                bad = ~((hi[l][k] == eh) & (lo[l][k] == el))
                assert not bad.any(), (ctx, "ema", l, k, int(bad.sum()), np.argwhere(bad)[:4].tolist())
        m[l] = mul32(add32(nh, -nl), gains[l])   # band_of: f32(f32(hi - lo) * gain)
    luma = prm["luma"]
    syn = slice(0, 1) if luma else slice(0, c)
    # the stored band: levels 1 and levels-1 (the others are the collapse's output on a frame that synthesises)
    # (a frame where every lane takes its first frame stores no band: the planes keep what they held)
    if not from_state:
        for l in band_levels:
            if l == 0 or (motion and 2 <= l <= lv - 2):
                continue
            for k in live:
                if all(o == "first" for o in ops):
                    if prev["band"].get(l) is not None:
                        assert np.array_equal(band[l][k], prev["band"][l][k]), (ctx, "band kept", l, k)
                    continue
                assert np.array_equal(band[l][k][syn], m[l][k][syn]), (ctx, "stored band", l, k)
                if luma and prev["band"].get(l) is not None:
                    assert np.array_equal(band[l][k][1:], prev["band"][l][k][1:]), (ctx, "a/b kept", l, k)
    else:
        for l in (1, lv - 1):
            if l >= 1 and not 2 <= l <= lv - 2:
                assert band[l] is None, (ctx, l)
    # the collapse
    cur = {lv - 1: m.get(lv - 1)}
    if motion:
        for l in range(lv - 2, 1, -1):
            fine_hw = Gd[l].shape[-2:]
            for k in live:
                ref = fma32(up_sum32(cur[l + 1][k][syn], fine_hw), INV64, m[l][k][syn])
                bad = band[l][k][syn] != ref
                assert not bad.any(), (ctx, "collapse", l, k, int(bad.sum()), np.argwhere(bad)[:4].tolist())
                if luma and prev["band"].get(l) is not None:
                    assert np.array_equal(band[l][k][1:], prev["band"][l][k][1:]), (ctx, "a/b kept", l, k)
            cur[l] = band[l]
    # the egress
    fout = hd.p.float_output(w, h, c)
    for k in live:
        if motion:
            if lv == 2:
                c1 = m[1][k][syn]
            else:
                c1 = fma32(up_sum32(cur[2][k][syn], Gd[1].shape[-2:]), INV64, m[1][k][syn])
            u = up_sum32(c1, (h, w))
        if c == 1:
            f = G0[k, 0]
            if motion:
                f = fma32(u[0], INV64, f)
            assert np.array_equal(fout[k, :, :, 0], f), (ctx, "egress gray", k)
            assert np.array_equal(out[k][:, :w], unit_to_u8(f)), (ctx, "egress gray u8", k)
            continue
        Lp, Ap, Bp = G0[k, 0], G0[k, 1], G0[k, 2]
        if motion:
            Lp = fma32(u[0], INV64, Lp)
            if not luma:
                ch64 = mul32(F32(prm["chroma"]), INV64)
                Ap = add32(Ap, mul32(u[1], ch64))
                Bp = add32(Bp, mul32(u[2], ch64))
        o = out[k][:, : 3 * w].reshape(h, w, 3)
        assert np.array_equal(o, unit_to_u8(fout[k])), (ctx, "egress u8", k)
        if prm.get("state_set"):
            # Lab' from state set to +-1e7 lies far outside any colour: there the egress's lg2 / ex2 approximations are
            # 2.1e-5 from cv2 (H100), beyond the 2e-5 the conversion meets on the Lab of real and perturbed colours
            continue
        ref = cv2.cvtColor(cv2.merge([Lp, Ap, Bp]), cv2.COLOR_Lab2BGR)
        err = float(np.abs(fout[k] - ref).max())
        stats["egress_float"] = max(stats["egress_float"], err)
        assert err <= FLOAT_TWIN_TOL, (ctx, "egress colour", k, err)
        d = np.abs(o.astype(np.int32) - unit_to_u8(ref).astype(np.int32))
        assert d.max() <= 1, (ctx, "egress u8 vs cv2", k)


# ---- content and the runner ------------------------------------------------------------------------------------------------
def frames_of(kind, t, lanes, w, h, c):
    if kind == "synth":
        f = np.stack([synth_frame(t, w, h, 3, seed=70 * k) for k in range(lanes)])
    else:
        f = np.stack([full_range_content(kind, t + 5 * k, w, h, seed=k) for k in range(lanes)])
    if c == 1:
        f = f[..., :1]
    return np.ascontiguousarray(f)


def run_laplace(w, h, c=3, lanes=1, levels=4, n=3, kind="noise", chroma=50, options=(), pad=0, events=None,
                co_low=None, co_high=None, set_state_at=None, seed=0, sensitivity=False):
    """n frame calls, every one checked stage by stage.  events[t]: [("restart", k) | ("hold", k, on)] before frame t;
    set_state_at: frame index before which every state plane is replaced by random values of both signs and large
    magnitude (mc_set_state).  -> stats (largest error / bound per bound kind)"""
    rng = np.random.default_rng(seed)
    lv = eff_levels(w, h, levels)
    opts = dict(options)
    faithful, from_state = opts.get("faithful_level0", 0) == 1, opts.get("band_from_state", 1) == 1
    hd, tw = Handle(lanes, options), Handle(lanes, options)
    stats = collections.Counter()
    stats["B"] = stats["B'"] = stats["egress_float"] = 0.0
    prm_p = params(levels, chroma=chroma, co_low=co_low, co_high=co_high)
    gains = gains_of(prm_p, lv, w, h)
    first, held = [True] * lanes, [False] * lanes
    ab_bounded = True
    groups = lane_groups(lanes, opts.get("lane_groups", 0))
    for t in range(n):
        for e in (events or {}).get(t, []):
            if e[0] == "restart":
                hd.p.restart_lane(e[1])
                first[e[1]] = True
            else:
                hd.p.hold_lane(e[1], e[2])
                held[e[1]] = bool(e[2])
        ops = ["hold" if held[k] else "first" if first[k] else "run" for k in range(lanes)]
        if set_state_at == t:
            for l in range(lv + 1):
                if hd.p.state_dims("lowpassHi", l)[0] > 0:
                    for nm in ("lowpassHi", "lowpassLo"):
                        a = hd.tap(nm, l)
                        v = rng.standard_normal(a.shape) * 10.0 ** rng.integers(-3, 7, a.shape)
                        hd.p.set_state(nm, l, v.astype(F32))
        prev = {"gauss": {l: hd.tap("gauss", l) for l in range(1, lv + 1)},
                "hi": {l: hd.tap("lowpassHi", l) for l in range(lv + 1)},
                "lo": {l: hd.tap("lowpassLo", l) for l in range(lv + 1)},
                "band": {l: hd.tap("band", l) for l in range(lv + 1)}}
        frames = frames_of(kind, t, lanes, w, h, c)
        c_lo = prm_p.coLow if prm_p.coLow != 0 else 0.01
        if "run" in ops and not (0 <= c_lo <= 1 and 0 <= prm_p.coHigh <= 1):
            ab_bounded = False
        luma = (c == 3 and opts.get("egress_strip", 1) == 1 and ab_bounded and F32(chroma) * INV64 == 0
                and all(abs(g) <= 2.0 ** 64 for g in gains))
        n0 = hd.p.launch_count
        produced, out = hd.frame(frames, prm_p, pad=pad)
        motion = "run" in ops and lv >= 2
        expect = 0 if all(o == "hold" for o in ops) else frame_launches(c, lv, ops, faithful, groups, motion)
        assert hd.p.launch_count - n0 == expect, (t, ops)
        assert bool(produced) == any(o != "hold" for o in ops), (t, ops)   # a first frame is converted
        tw.p.reset()
        tw.frame(frames, prm_p, pad=pad)
        prm = dict(lv=lv, faithful=faithful, from_state=from_state, co_high=prm_p.coHigh, co_low=prm_p.coLow,
                   gains=gains, luma=luma, chroma=prm_p.chromAttenuation, sensitivity=sensitivity,
                   state_set=set_state_at is not None and t >= set_state_at)
        check_frame(hd, tw, frames, out, ops, prev, prm, stats, (w, h, c, lanes, t))
        for k in range(lanes):
            first[k] = first[k] and held[k]
    hd.close()
    tw.close()
    for key in ("B", "B'", "egress_float"):
        SEEN[key] = max(SEEN[key], stats[key])
    return stats


# ---- the sweep -------------------------------------------------------------------------------------------------------------
# Widths at the 120-column strip seams of k_ingest_lab / k_down_strip / the strip egress (121, 241, 361), around the 64 x 32
# level tile (65, 129, 193), an exact tile (128 x 64: pitch == width), sizes odd at every level (257 x 129 -> 9 x 5),
# the ingest's 32 coarse rows per warp (65, 129 rows) and k_down_strip's 16 x 4 row chunk, EG_ROWS = 64 (65, 129 rows),
# widths of every residue mod 4 (word / byte stores), and the smallest sizes the level clamp allows.
SWEEP = [
    # w,   h,  c, lanes, levels, options, pad, kind
    (121, 33, 3, 1, 3, (), 0, "noise"),
    (241, 65, 1, 1, 4, (), 0, "noise"),
    (361, 70, 3, 3, 5, (("lane_groups", 2),), 0, "checker"),
    (128, 64, 3, 1, 4, (("use_tma", 0),), 0, "blocks"),
    (128, 64, 1, 3, 4, (("band_from_state", 0),), 0, "noise"),
    (257, 129, 3, 1, 8, (), 0, "noise"),
    (257, 129, 1, 1, 8, (("use_tma", 0), ("band_from_state", 0)), 0, "shadows"),
    (130, 66, 3, 1, 2, (("egress_strip", 0),), 0, "noise"),
    (131, 131, 3, 3, 3, (("band_from_state", 0), ("lane_groups", 2)), 3, "synth"),
    (193, 97, 1, 1, 5, (("egress_strip", 0),), 1, "checker"),
    (6, 6, 3, 1, 8, (), 0, "noise"),
    (11, 7, 1, 1, 8, (), 0, "noise"),
    (67, 41, 3, 1, 4, (("faithful_level0", 1),), 0, "noise"),
    (66, 35, 1, 1, 3, (("faithful_level0", 1), ("band_from_state", 0)), 2, "blocks"),
    (129, 65, 3, 1, 1, (), 0, "noise"),
    (9, 9, 3, 1, 1, (("faithful_level0", 1),), 0, "noise"),
]


@pytest.mark.parametrize("w,h,c,lanes,levels,options,pad,kind", SWEEP)
@pytest.mark.parametrize("chroma", [50, 0])
def test_every_stage_on_the_seam_sweep(w, h, c, lanes, levels, options, pad, kind, chroma):
    assert {x % 4 for x, *_ in SWEEP} == {0, 1, 2, 3}
    s = run_laplace(w, h, c, lanes, levels, n=3, kind=kind, chroma=chroma, options=options, pad=pad,
                    seed=w * 1000 + h, sensitivity=kind == "noise")
    if "sens0" in s:   # noise content, G_1 built
        assert s["sens0"] >= 2 ** 10, s   # a wrong tap or border source of the ingest / down strip is >= 2^10 bounds off


@pytest.mark.parametrize("tma", [0, 1])
@pytest.mark.parametrize("c", [1, 3])
def test_ema_bit_for_bit_with_state_set_and_extreme_cutoffs(tma, c):
    """The EMA from state planes of both signs and magnitudes up to about 1e7 (mc_set_state): coLow 0 (the driver takes 0.01),
    coHigh above 1 (which also clears the L-only synthesis), and ordinary cutoffs"""
    for co_low, co_high in ((0.0, 0.7), (0.05, 1.5), (0.3, 0.9)):
        run_laplace(133, 70, c, 1, 4, n=3, set_state_at=1, co_low=co_low, co_high=co_high,
                    options=(("use_tma", tma),), seed=int(co_high * 10))


@pytest.mark.parametrize("kind", ["synth", "noise", "checker", "blocks", "shadows"])
def test_every_stage_on_full_range_content(kind):
    run_laplace(241, 97, 3, 1, 5, n=3, kind=kind)


def test_lanes_run_first_and_hold_in_one_frame():
    """3 lanes: lane 1 restarted at frame 2 (FIRST while lane 0 runs), lane 2 held over frames 2-3 (pyramid, state,
    band planes and output bytes unchanged), then all run"""
    events = {2: [("restart", 1), ("hold", 2, 1)], 4: [("hold", 2, 0)]}
    for opts in ((), (("band_from_state", 0), ("use_tma", 0))):
        run_laplace(135, 66, 3, 3, 4, n=5, events=events, options=opts)
    run_laplace(135, 66, 1, 3, 3, n=5, events=events, options=(("lane_groups", 2),))


@pytest.mark.skipif(EMU, reason="full-HD frames are too slow for the CPU emulation")
def test_every_stage_on_a_1080p_frame():
    run_laplace(1920, 1080, 3, 1, 6, n=2, kind="synth")


def test_taps_are_read_only_and_absent_without_a_frame():
    hd = Handle(2)
    p = params(3)
    f = frames_of("noise", 0, 2, 40, 24, 3)
    assert hd.p.state_dims("gauss", 1) == (0, 0, 0)
    n0 = hd.p.launch_count
    hd.frame(f, p)
    assert hd.p.launch_count - n0 == 1 + 2 + 1   # ingest_lab, level 1, level 2, egress
    for l in (1, 2, 3):
        a = hd.tap("gauss", l)
        assert a is not None and a.shape == (2, 3, (24 + 2 ** l - 1) >> l, (40 + 2 ** l - 1) >> l)
        with pytest.raises(L.MagcoreError) as e:
            hd.p.set_state("gauss", l, a)
        assert e.value.status == capi.MC_ERR_INVALID
    assert hd.p.state_dims("gauss", 0) == (0, 0, 0) and hd.p.state_dims("gauss", 4) == (0, 0, 0)
    hd.p.reset()
    assert hd.p.state_dims("gauss", 1) == (0, 0, 0)
    hd.frame(f, p)
    assert hd.p.state_dims("gauss", 1) == (12, 20, 3)
    hd.p.process_clip(np.stack([f, f]), make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 50, 3, 30.0)[0])
    assert hd.p.state_dims("gauss", 1) == (0, 0, 0)               # a clip call: its pyramid is the clip's own
    hd.frame(f, p)
    assert hd.p.state_dims("gauss", 1) == (12, 20, 3)
    hd.frame(frames_of("noise", 1, 2, 48, 24, 3), p)              # new geometry: a first frame
    assert hd.p.state_dims("gauss", 1) == (12, 24, 3)
    hd.frame(frames_of("noise", 2, 2, 48, 24, 1), p)              # gray input: the tap exists too
    assert hd.p.state_dims("gauss", 1) == (12, 24, 1)
    hd.frame(frames_of("noise", 2, 2, 48, 24, 3), make_cfgs(O.MODE_PHASE, 50, 50.0, 0.4, 3.0, 0, 3, 30.0)[0])
    assert hd.p.state_dims("gauss", 1) == (0, 0, 0)               # another mode
    hd.close()
    one = Handle(1)
    one.frame(frames_of("noise", 0, 1, 40, 24, 3), params(1))
    assert one.p.state_dims("gauss", 1) == (0, 0, 0)              # one level: no kernel builds G_1
    one.close()
