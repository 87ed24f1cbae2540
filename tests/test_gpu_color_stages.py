"""Color mode stage by stage, through the read-only taps "gauss", "window", "filtered" and "up" (mc_get_state).

Every stage is teacher-forced: its reference is computed on the host from the device's own previous tap, so each
comparison isolates one kernel and the tolerance is that kernel's own:

  ingest            gauss[0] == float(u8), exactly
  k_down_strip      gauss[l+1] vs a float64 5x5 [1 4 6 4 1]^2 / 256 with reflect-101 borders of gauss[l]: exactly at
                    l = 0, 1 (every partial sum is an integer below 2^24 over a power of two, so any evaluation order
                    gives the same bits), <= 4 ulp deeper (f32 partial sums in the row and in the column pass, whose contraction
                    to FMAs is the compiler's; 2.02 ulp measured on the CPU emulation)
  ring              window[k] == the gauss[levels] taps of the last n frames, bit for bit, in order
  cuFFT + mask      filtered vs a float64 DFT -> complex CCS mask -> inverse: <= 1e-5 of the window's range
  k_minmax/k_select up[0] == fmaf(filtered[1], 1/(max-min), -min/(max-min)) * alpha from the downloaded columns, bit for bit
  k_pyrup2x         up[i+1] == the kernel's _rn-pinned taps evaluated on up[i], bit for bit
  k_resize_linear   vs a float64 bilinear with the f32 coefficients of cv::resize: <= 2^-21 of the plane's largest magnitude
                    (1.2 * 2^-23 measured on the CPU emulation); vs cv2.resize(INTER_LINEAR) itself <= 2^-18: cv2 is
                    not bit-equal and is the less accurate of the two (10 * 2^-23 off the float64 result at a ratio
                    just below 1); a wrong source pixel is off by a gradient, 1e-3 or more
  k_sum_minmax      the u8 output == convertTo(gauss[0] + up[last], 255/(max-min), -min*255/(max-min)) on the host,
  + egress          byte for byte

The level clamp of the API (both sides of a level that is halved exceed 5 pixels) keeps the smallest level at 3 pixels or
more a side, so frames start at 6 pixels and the sweep takes every level down to 3 x k."""
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O
from common import make_cfgs, planar, u8_diff
import np_model as M

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
EMU = os.environ.get("MC_EMU") == "1"
LIFECYCLE = (("color_lane_lifecycle", 1),)


def eff_levels(w, h, levels):
    return min(max(levels, 1), O.calculate_max_levels(w, h))


class Handle:
    """A Color handle fed [lanes][h][w][c] u8 frames (optionally with padded rows), with its taps."""

    def __init__(self, lanes=1, options=()):
        self.p = L.MagnificationProcessor(0, lanes=lanes)
        self.p.set_option("keep_float_output", 1)
        for k, v in options:
            self.p.set_option(k, v)
        self.lanes = lanes

    def frame(self, frames, cfg, pad=0):
        lanes, h, w, c = frames.shape
        assert lanes == self.lanes
        step = w * c + pad
        buf = np.full((lanes, h, step), 0xEE, np.uint8)
        buf[:, :, :w * c] = frames.reshape(lanes, h, w * c)
        out = np.zeros_like(buf)
        produced = self.p.process_host(buf.ctypes.data, w, h, c, step, cfg, out.ctypes.data, step)
        return produced, out[:, :, :w * c].reshape(frames.shape)

    def tap(self, name, level=0):
        return self.p.get_state(name, level)

    def columns(self, name):
        n = 0
        while self.p.state_dims(name, n)[0] > 0:
            n += 1
        return n

    def close(self):
        self.p.close()


# ---- host references ---------------------------------------------------------------------------------------------------
def pyr_down64(p):
    """float64 cv::pyrDown of [..., h, w] planes"""
    h, w = p.shape[-2:]
    xs = [M.reflect101(2 * np.arange((w + 1) // 2) + d, w) for d in (-2, -1, 0, 1, 2)]
    row = 6 * p[..., xs[2]] + 4 * (p[..., xs[1]] + p[..., xs[3]]) + p[..., xs[0]] + p[..., xs[4]]
    ys = [M.reflect101(2 * np.arange((h + 1) // 2) + d, h) for d in (-2, -1, 0, 1, 2)]
    return (6 * row[..., ys[2], :] + 4 * (row[..., ys[1], :] + row[..., ys[3], :]) + row[..., ys[0], :] + row[..., ys[4], :]) / 256


def fma32(a, b, c):
    """f32 fmaf(a, b, c): the product of two f32 is exact in float64; the sum is rounded there once more, which changes
    the f32 result only on a tie of about 2^-29 probability per element"""
    return (a.astype(F64) * F64(b) + np.asarray(c, F32).astype(F64)).astype(F32)


def pyr_up_exact(p):
    """k_pyrup2x's arithmetic on [..., h, w] f32 planes -> [..., 2h, 2w]: even taps fmaf(s[i], 6, s[i-1]) + s[i+1], odd
    taps (s[i] + s[i+1]) * 4, rows then columns, / 64; s[-1] := s[1], s[n] := s[n-1]"""
    def taps(s, axis):
        s = np.moveaxis(s, axis, -1)
        n = s.shape[-1]
        i = np.arange(n)
        sm1, sp1 = s[..., np.where(i == 0, 1, i - 1)], s[..., np.minimum(i + 1, n - 1)]
        even = (fma32(s, 6.0, sm1) + sp1).astype(F32)
        odd = ((s + sp1).astype(F32) * F32(4)).astype(F32)
        out = np.stack([even, odd], axis=-1).reshape(s.shape[:-1] + (2 * n,))
        return np.moveaxis(out, -1, axis)
    return (taps(taps(p.astype(F32), -1), -2) * F32(1 / 64)).astype(F32)


def resize64(s, w, h):
    """cv::resize(INTER_LINEAR) of one [sh][sw] plane to h x w in float64, with the f32 coefficients the reference and the
    kernel both take: f = (float)((x + 0.5) * sw / w - 0.5), split into floor and fraction, clamped at both ends"""
    def coef(n_d, n_s):
        f = ((np.arange(n_d) + 0.5) * (F64(n_s) / n_d) - 0.5).astype(F32)
        i = np.floor(f).astype(int)
        f = (f - i.astype(F32)).astype(F32)
        f, i = np.where(i < 0, 0, f), np.maximum(i, 0)
        f, i = np.where(i >= n_s - 1, 0, f), np.minimum(i, n_s - 1)
        return i, np.minimum(i + 1, n_s - 1), f.astype(F64)
    (x0, x1, fx), (y0, y1, fy) = coef(w, s.shape[1]), coef(h, s.shape[0])
    r = s.astype(F64)[:, x0] * (1 - fx) + s.astype(F64)[:, x1] * fx
    return r[y0] * (1 - fy)[:, None] + r[y1] * fy[:, None]


def filter64(win, lo, hi, fps):
    """The reference's idealFilter before its normalisation, in float64, on [n, ...] columns: DFT_SCALE forward, the 0/1
    mask over PACKED indices read back as mulSpectrums reads it (m[2k-1] + i m[2k]; real for DC and Nyquist), DFT_SCALE
    inverse"""
    n = win.shape[0]
    m = O.create_ideal_bandpass_filter(1, n, lo if lo != 0.0 else 0.01, hi, fps)[0].astype(F64)
    k = np.arange(n // 2 + 1)
    cm = np.where(k == 0, m[0], m[np.maximum(2 * k - 1, 0)] + 1j * m[np.minimum(2 * k, n - 1)])
    if n % 2 == 0:
        cm[-1] = m[n - 1]
    spec = np.fft.rfft(win.astype(F64), axis=0) / n
    return np.fft.irfft(spec * cm.reshape((-1,) + (1,) * (win.ndim - 1)), n=n, axis=0), m


def select_exact(filt, alpha):
    """k_minmax + k_select on one lane's filtered columns [n, c, h, w] -> up[0] [c, h, w]"""
    mn, mx = F64(filt.min()), F64(filt.max())
    scale = 1.0 / (mx - mn) if mx - mn > np.finfo(F64).eps else 0.0
    shift = 0.0 - mn * scale
    return (fma32(filt[min(1, len(filt) - 1)], F32(scale), F32(shift)) * F32(alpha)).astype(F32)


def stretch_exact(v):
    """the output stretch of one lane's f32 image (any layout) -> u8, as convertTo evaluates it"""
    mn, mx = F64(v.min()), F64(v.max())
    with np.errstate(all="ignore"):
        sa, sb = F32(F64(255.0) / (mx - mn)), F32(-mn * 255.0 / (mx - mn))
        r = np.rint(fma32(v, sa, sb).astype(F64))
    r = np.where(~np.isfinite(r) | (r >= 2147483648.0) | (r < -2147483648.0), -2147483648.0, r)
    return np.clip(r, 0, 255).astype(np.uint8)


def ulps(got, ref64):
    return np.abs(got.astype(F64) - ref64) / np.spacing(np.maximum(np.abs(ref64), 1e-30).astype(F32)).astype(F64)


# ---- the stage checkers (shared with tests/test_emu_color_stages.py) -------------------------------------------------------
def check_gauss(hd, frames, levels):
    g = [hd.tap("gauss", l) for l in range(levels + 1)]
    assert hd.tap("gauss", levels + 1) is None
    assert np.array_equal(g[0], frames.transpose(0, 3, 1, 2).astype(F32))
    for l in range(levels):
        ref = pyr_down64(g[l].astype(F64))
        assert g[l + 1].shape == ref.shape, l
        if l < 2:
            assert np.array_equal(g[l + 1], ref), l
        else:
            assert ulps(g[l + 1], ref).max() <= 4, (l, ulps(g[l + 1], ref).max())
    return g


def check_filter(hd, lo, hi, fps):
    """-> (window, filtered) as [lanes][n][c][h][w]"""
    n = hd.columns("window")
    assert hd.columns("filtered") == n >= 2
    win = np.stack([hd.tap("window", k) for k in range(n)], axis=1)
    filt = np.stack([hd.tap("filtered", k) for k in range(n)], axis=1)
    for lane in range(hd.lanes):
        ref, mask = filter64(win[lane], lo, hi, fps)
        rng = float(win[lane].max() - win[lane].min())
        err = float(np.abs(filt[lane] - ref).max())
        assert err <= 1e-5 * rng, (lane, n, err, rng)
        assert filt[lane].any() == mask.any()   # a band that keeps nothing: exactly zero; otherwise the later stages see data
    return win, filt


def check_synthesis(hd, frames, out, levels, alpha, filt, g0):
    """select, pyrUp chain, resize, output sum and stretch of the last frame call"""
    lanes, h, w, c = frames.shape
    up = [hd.tap("up", i) for i in range(levels + 1)]
    for lane in range(lanes):
        assert np.array_equal(up[0][lane], select_exact(filt[lane], alpha)), lane
    for i in range(levels):
        assert np.array_equal(up[i + 1], pyr_up_exact(up[i])), i
    color = up[levels]
    resized = hd.tap("up", levels + 1)
    assert (resized is not None) == (color.shape[2:] != (h, w))
    assert hd.tap("up", levels + 2) is None
    if resized is not None:
        for pl, src in zip(resized.reshape(-1, h, w), color.reshape((-1,) + color.shape[2:])):
            mag = max(float(np.abs(src).max()), 1e-30)
            assert np.abs(pl - resize64(src, w, h)).max() <= mag * 2.0 ** -21
            assert np.abs(pl - cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR)).max() <= mag * 2.0 ** -18
        color = resized
    total = (g0 + color).astype(F32)                            # input + colour image, one f32 add
    got = hd.p.float_output(w, h, c)
    assert np.array_equal(got, total.transpose(0, 2, 3, 1))
    for lane in range(lanes):
        assert np.array_equal(out[lane], stretch_exact(got[lane])), (lane, int(u8_diff(out[lane], stretch_exact(got[lane])).max()))
    return up


def check_frame(hd, frames, out, levels, alpha, lo, hi, fps):
    """Every stage of the frame call that just produced `out`, each from the device's own previous tap"""
    g = check_gauss(hd, frames, levels)
    win, filt = check_filter(hd, lo, hi, fps)
    assert np.array_equal(win[:, -1], g[levels])
    check_synthesis(hd, frames, out, levels, alpha, filt, g[0])
    return g, win, filt


def noise_frames(rng, lanes, h, w, c, kind="noise", base=None):
    """one [lanes][h][w][c] frame of the content kinds tests/tools/fuzz_parity.py draws: full-range noise, saturated with
    dither, impulses"""
    shape = (lanes, h, w, c)
    if kind == "noise":
        f = rng.integers(0, 256, size=shape)
    elif kind == "saturated":
        f = np.where(base > 128, 255, 0) + rng.integers(-1, 2, size=shape)
    else:
        f = np.full(shape, 20)
        f.reshape(lanes, h * w, c)[:, rng.integers(0, h * w, size=max(1, h * w // 50))] = 250
        f = f + rng.integers(0, 2, size=shape)
    return np.clip(f, 0, 255).astype(np.uint8)


def run_stages(w, h, c, lanes, levels=8, n=3, fps=8.0, lo=0.5, hi=4.0, alpha=100, pad=0, seed=0, kind="noise", oracle=False):
    """n frames through a handle, every produced frame checked stage by stage (and, with `oracle`, free-running against
    the oracle at the end-to-end tolerance).  The default band, 0.5-4 Hz at 8 fps, keeps bins of a 2- and a 3-column
    window, so the stages after the filter see data from the first produced frame on."""
    rng = np.random.default_rng(seed)
    lv = eff_levels(w, h, levels)
    cfg, ocfg = make_cfgs(O.MODE_COLOR, alpha, 0.0, lo, hi, 0, levels, fps)
    hd = Handle(lanes)
    oprocs = [O.MagnificationProcessor() for _ in range(lanes if oracle else 0)]
    base = rng.integers(0, 256, size=(lanes, h, w, c))
    launches = []
    for t in range(n):
        frames = noise_frames(rng, lanes, h, w, c, kind, base)
        before = hd.p.launch_count
        produced, out = hd.frame(frames, cfg, pad)
        launches.append(hd.p.launch_count - before)
        assert produced == (t > 0)
        for k, op in enumerate(oprocs):
            dbg = {}
            oprod, oout = op.process(frames[k] if c == 3 else frames[k, ..., 0], ocfg, dbg)
            assert oprod == produced
            if produced:
                ref = dbg["output_f32"].reshape(h, w, c)
                # dithered static content moves the window by a few 1e-2 only: the normalisation magnifies the f32
                # rounding of the two pyramids by 1 / that range, so the float tolerance is for noise (the stages below are
                # checked on every kind)
                assert kind != "noise" or np.abs(hd.p.float_output(w, h, c)[k] - ref).max() / 255.0 < 1e-4
                assert int(u8_diff(out[k], oout.reshape(h, w, c)).max()) <= 1
        if produced:
            check_frame(hd, frames, out, lv, alpha, lo, hi, fps)
        else:
            check_gauss(hd, frames, lv)
            assert hd.columns("window") == 1 and hd.columns("filtered") == 0 and hd.tap("up", 0) is None
    hd.close()
    return launches


# widths and heights around the kernels' seams: k_down_strip's 120-column strips and 32-lane halos, k_pyrup2x's 64 x 32
# tiles, the 4-wide vectors of the reductions; 6 is the smallest side the API magnifies
SEAMS = [6, 7, 9, 11, 31, 32, 33, 63, 64, 65, 119, 120, 121, 124, 128, 129, 240, 241, 255, 257]
SWEEP = [(SEAMS[i], SEAMS[(i + 7) % len(SEAMS)], (1, 3)[i % 2], (1, 3)[(i // 2) % 2]) for i in range(len(SEAMS))]
KINDS = ("noise", "saturated", "impulses")


@pytest.mark.parametrize("w,h,c,lanes", SWEEP)
def test_every_stage_on_the_seam_sweep(w, h, c, lanes):
    """Deepest pyramid the size allows, full-range noise, padded input rows; stage by stage and against the oracle."""
    run_stages(w, h, c, lanes, pad=5, seed=w * 1000 + h, oracle=True)


@pytest.mark.parametrize("w,h,c,lanes", SWEEP[::3])
@pytest.mark.parametrize("kind", KINDS[1:])
def test_seam_sweep_on_saturated_and_impulse_content(w, h, c, lanes, kind):
    run_stages(w, h, c, lanes, seed=w + h, kind=kind, oracle=True)


def test_resize_for_every_excess_of_the_pyrup_chain():
    """levels 3: the chain ends at 8 * ceil(side / 8); every excess 1..7 in width and in height, the ratios just below 1
    and the clamps at the last source column and row"""
    for k in range(1, 8):
        w, h = 64 - k, 40 + k
        assert eff_levels(w, h, 3) == 3
        run_stages(w, h, 3, 1, levels=3, n=2, seed=k)


def test_taps_do_not_change_the_launch_count_of_a_frame():
    """ingest + 2 pyrDown + append = 4 launches while warming; + R2C, mask, C2R, min/max init, min/max, select, 2 pyrUp,
    resize, output min/max, egress = 15 per produced frame — reading taps in between adds none"""
    assert run_stages(91, 67, 3, 3, levels=2, n=4) == [4, 15, 15, 15]


def test_taps_are_read_only_and_absent_without_a_frame():
    hd = Handle(2)
    cfg = make_cfgs(O.MODE_COLOR, 100, 0.0, 0.8, 1.2, 0, 2, 8.0)[0]
    names = ("gauss", "window", "filtered", "up")
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in names)
    rng = np.random.default_rng(1)
    for _ in range(2):
        hd.frame(noise_frames(rng, 2, 24, 40, 3), cfg)
    for nm in names:
        a = hd.tap(nm, 0)
        assert a is not None and a.shape[:2] == (2, 3)
        with pytest.raises(L.MagcoreError) as e:
            hd.p.set_state(nm, 0, a)
        assert e.value.status == capi.MC_ERR_INVALID
    hd.p.reset()
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in names)
    hd.frame(noise_frames(rng, 2, 24, 40, 3), cfg)
    hd.frame(noise_frames(rng, 2, 24, 40, 3), cfg)
    assert hd.tap("up", 0) is not None
    hd.frame(noise_frames(rng, 2, 24, 48, 3), cfg)            # structural change: a fresh one-column window
    assert hd.columns("window") == 1 and hd.tap("up", 0) is None
    hd.frame(noise_frames(rng, 2, 24, 48, 3), make_cfgs(O.MODE_NONE, 100, 0.0, 0.8, 1.2, 0, 2, 8.0)[0])
    assert all(hd.p.state_dims(nm, 0) == (0, 0, 0) for nm in names)
    hd.close()


# ---- the window ------------------------------------------------------------------------------------------------------------
def drive_window(w, h, c, lanes, script, levels=2, events=None, options=()):
    """script: fps per frame.  After every frame window[k] of every lane must be, bit for bit and in order, the
    gauss[levels] taps of the frames the lane appended, cut to the length the reference's window has; lanes in lock-step
    are also checked stage by stage.  events[t]: [("restart", k) | ("hold", k, on)] before frame t."""
    rng = np.random.default_rng(w * h + lanes)
    lv = eff_levels(w, h, levels)
    hd = Handle(lanes, options)
    oprocs = [O.MagnificationProcessor() for _ in range(lanes)]
    hist = [[] for _ in range(lanes)]
    held = [False] * lanes
    for t, fps in enumerate(script):
        for e in (events or {}).get(t, []):
            if e[0] == "hold":
                hd.p.hold_lane(e[1], e[2])
                held[e[1]] = bool(e[2])
            else:
                hd.p.restart_lane(e[1])
                oprocs[e[1]].reset()
                hist[e[1]] = []
        cfg, ocfg = make_cfgs(O.MODE_COLOR, 100, 0.0, 0.8, 1.2, 0, levels, fps)
        frames = noise_frames(rng, lanes, h, w, c)
        produced, out = hd.frame(frames, cfg)
        small = hd.tap("gauss", lv)
        for k in range(lanes):
            if held[k]:
                continue
            oprocs[k].process(frames[k] if c == 3 else frames[k, ..., 0], ocfg)
            hist[k] = (hist[k] + [small[k]])[-oprocs[k].color.window.shape[1]:]   # the reference's length rule
        n = hd.columns("window")
        assert n == min(len(x) for x in hist), t                  # a column is served while every lane has it
        for j in range(n):
            col = hd.tap("window", j)
            for k in range(lanes):
                assert np.array_equal(col[k], hist[k][j]), (t, j, k)
                ocol = planar(oprocs[k].color.window[:, j].reshape(small.shape[2], small.shape[3], c))
                assert np.abs(col[k] - ocol).max() < 1e-3, (t, j, k)
        if produced and len({len(x) for x in hist}) == 1 and not any(held):
            check_frame(hd, frames, out, lv, 100, 0.8, 1.2, fps)
    hd.close()


@pytest.mark.parametrize("c,lanes", [(3, 1), (1, 3)])
def test_window_through_warmup_wrap_and_framerate_changes(c, lanes):
    """cap 16 warm-up and wrap (21 frames), 8 -> 30 (grow to 64 while full) -> 8 (a longer window keeps its length) -> 7
    fps.  1 channel x 3 lanes of 23 x 17 small pixels: odd lane blocks, the padding float in play."""
    drive_window(91, 67, c, lanes, [8.0] * 21 + [30.0] * 9 + [8.0] * 5 + [7.0] * 4)


def test_window_shrinks_while_partly_filled():
    drive_window(40, 30, 3, 1, [30.0] * 20 + [8.0] * 20 + [30.0] * 3)


def test_window_per_lane_restart_and_hold():
    """3 lanes of 3 x 23 x 17 signals (odd: padded): a restart in warm-up and one after the wrap, a hold across the wrap"""
    events = {5: [("restart", 1)], 9: [("hold", 2, 1)], 19: [("hold", 2, 0)], 24: [("restart", 0)]}
    drive_window(91, 67, 3, 3, [8.0] * 30, events=events, options=LIFECYCLE)


# ---- the temporal filter -------------------------------------------------------------------------------------------------
def test_filter_every_window_length_2_to_64():
    """30 fps: cap 64; every warm-up length, odd ones included, and 3 wrapped frames"""
    assert run_stages(33, 24, 3, 1, levels=2, n=67, fps=30.0, lo=0.8, hi=1.2) == [4] + [15] * 66


# (fps, low, high): at 8 fps the packed index of a frequency f is 2 f n / 8 = f n / 4
MASKS = [
    (8.0, 1.0, 2.0),      # n = 4k: both edges land on packed indices exactly (n = 16: fl = 4, fh = 8), inclusive
    (8.0, 0.0, 0.5),      # low 0 -> 0.01 Hz: DC stays out, n = 16: fh = 2
    (8.0, 0.0, 4.0),      # up to Nyquist: the real Nyquist bin of even n (packed index n - 1) and of odd n
    (8.0, 3.9, 4.0),      # the last packed indices only
    (8.0, 1.2, 0.8),      # fl > fh: keeps nothing
    (8.0, 0.26, 0.27),    # between two packed indices for most n: keeps nothing
    (8.0, 0.5, 0.5),      # one packed index when n is a multiple of 8: a real part or an imaginary part alone
]


@pytest.mark.parametrize("fps,lo,hi", MASKS)
def test_filter_mask_cases(fps, lo, hi):
    run_stages(24, 40, 3, 2, levels=2, n=19, fps=fps, lo=lo, hi=hi, seed=5, oracle=True)


# ---- reductions with the extremum where a kernel could drop it --------------------------------------------------------
def flicker_case(w, h, c, lanes, levels, n, lane, ch, y, x, slot, sign):
    """A static noise frame per lane plus a temporal flicker under small-level pixel (y, x) of channel ch: the filtered
    window's maximum (sign +1) or minimum (-1) of `lane` must sit exactly there, in time slot `slot`; other lanes flicker
    elsewhere and weaker.  Asserts the place from the tap, then checks every stage."""
    lv = eff_levels(w, h, levels)
    assert lv == levels
    fps, lo, hi = 8.0, 0.8, 1.2
    resp = filter64(np.eye(n), lo, hi, fps)[0][:, 0]             # response to an impulse at t = 0; shifts with the impulse
    t0 = (slot - int(np.argmax(resp))) % n
    rng = np.random.default_rng(7)
    base = rng.integers(96, 160, size=(lanes, h, w, c))
    cfg = make_cfgs(O.MODE_COLOR, 100, 0.0, lo, hi, 0, levels, fps)[0]
    hd = Handle(lanes)
    r = 1 << (levels - 1)

    def bump(f, k, cy, cx, cc, a):
        f[k, max(cy * 2 * r - r, 0):cy * 2 * r + r + 1, max(cx * 2 * r - r, 0):cx * 2 * r + r + 1, cc] += a

    sh, sw = hd_small = ((h + (1 << levels) - 1) >> levels, (w + (1 << levels) - 1) >> levels)
    for t in range(n):
        f = base.copy()
        if t == t0:
            for k in range(lanes):
                if k == lane:
                    bump(f, k, y, x, ch, 90 * sign)
                else:
                    bump(f, k, sh // 2, sw // 2, 0, 40 * sign)
        frames = np.clip(f, 0, 255).astype(np.uint8)
        produced, out = hd.frame(frames, cfg)
    g, win, filt = check_frame(hd, frames, out, lv, 100, lo, hi, fps)
    assert win.shape[1:] == (n, c, sh, sw), (win.shape, hd_small)
    at = np.unravel_index(np.argmax(sign * filt[lane]), filt[lane].shape)
    assert at == (slot, ch, y, x), (at, (slot, ch, y, x))
    hd.close()


# (w, h, c, lanes, levels): channels * small pixels per lane, and what it selects in k_minmax
#   (24, 16, 3, 1, 1)  12 x 8 x 3 = 288: vector path, one CTA
#   (44, 30, 3, 1, 1)  22 x 15 x 3 = 990: scalar path (990 = 2 mod 4), one CTA
#   (46, 30, 3, 1, 1)  23 x 15 x 3 = 1035: scalar path (3 mod 4), two CTAs (past 1024)
#   (26, 26, 1, 1, 1)  13 x 13 = 169: scalar path (1 mod 4)
#   (64, 48, 3, 2, 1)  32 x 24 x 3 = 2304: vector path, three CTAs, two lanes
#   (46, 30, 1, 5, 1)  23 x 15 = 345 (odd: padded lanes, scalar path), five lanes
GEOMS = [(24, 16, 3, 1, 1), (44, 30, 3, 1, 1), (46, 30, 3, 1, 1), (26, 26, 1, 1, 1), (64, 48, 3, 2, 1), (46, 30, 1, 5, 1)]


@pytest.mark.parametrize("sign", [1, -1])
@pytest.mark.parametrize("w,h,c,lanes,levels", GEOMS)
def test_extremum_in_the_last_element_last_channel_last_slot_last_lane(w, h, c, lanes, levels, sign):
    sh, sw = (h + 1) // 2, (w + 1) // 2
    flicker_case(w, h, c, lanes, levels, 7, lanes - 1, c - 1, sh - 1, sw - 1, 6, sign)


@pytest.mark.parametrize("sign", [1, -1])
@pytest.mark.parametrize("w,h,c,lanes,levels", GEOMS[:2] + GEOMS[4:])
def test_extremum_in_the_first_element_first_slot(w, h, c, lanes, levels, sign):
    flicker_case(w, h, c, lanes, levels, 5, lanes - 1, 0, 0, 0, 0, sign)


@pytest.mark.parametrize("back", [1, 2, 3])
def test_extremum_in_the_last_vector_of_a_chunk(back):
    """288 floats a lane: the maximum in the last 128-bit vector, 1..3 elements before the end"""
    flicker_case(24, 16, 3, 1, 1, 5, 0, 2, 7, 11 - back, 4, 1)


@pytest.mark.skipif(EMU, reason="70 lanes are too slow for the CPU emulation")
@pytest.mark.parametrize("w,h", [(64, 48), (128, 96)])
def test_extremum_in_the_last_lane_of_70(w, h):
    """70 lanes: 9 CTAs a lane at most.  64 x 48: 2304 floats a lane, 3 CTAs; 128 x 96: 9216 floats, the cap of 9 (below
    9216 / 1024 + 1) is in force and each thread strides"""
    flicker_case(w, h, 3, 70, 1, 4, 69, 2, h // 2 - 1, w // 2 - 1, 3, 1)
    flicker_case(w, h, 3, 70, 1, 4, 69, 2, h // 2 - 1, w // 2 - 1, 3, -1)


# ---- the output stretch, exactly -----------------------------------------------------------------------------------------
def stretch_case(w, h, c, lanes, lane, lo_at, hi_at):
    """Amplification 0: the colour image is +-0 and the output is the contrast stretch of the input.  Mid-grey frames with
    one pixel of 3 at lo_at and one of 250 at hi_at ((y, x, channel)) in `lane`, 40 / 200 at the centre of the others."""
    cfg, ocfg = make_cfgs(O.MODE_COLOR, 0, 0.0, 0.8, 1.2, 0, 1, 8.0)
    frames = np.full((lanes, h, w, c), 128, np.uint8)
    frames[:, h // 2, w // 2, 0], frames[:, h // 2, w // 2 + 1, 0] = 40, 200
    frames[lane][lo_at], frames[lane][hi_at] = 3, 250
    hd, op = Handle(lanes), O.MagnificationProcessor()
    for t in range(2):
        f = frames.copy()
        f[:, 0, w // 2, 0] = 100 + 20 * t                          # a window that is not constant in time
        produced, out = hd.frame(f, cfg)
        _, oout = op.process(f[lane] if c == 3 else f[lane, ..., 0], ocfg)
    assert produced
    assert not hd.tap("up", 1).any()
    v = f[lane].astype(F64)
    want = np.clip(np.rint(((v - 3) * 255 / 247).astype(F32)), 0, 255).astype(np.uint8)   # 3 -> 0, 250 -> 255
    assert int(u8_diff(out[lane], want).max()) <= 1              # the plain-arithmetic sanity of the two exact checks below
    assert np.array_equal(out[lane], stretch_exact(f[lane].astype(F32)))
    assert np.array_equal(out[lane], oout.reshape(h, w, c))
    other = stretch_exact(f[0].astype(F32))
    if lane != 0:
        assert np.array_equal(out[0], other) and out[0].max() == 255 and out[0].min() == 0
    hd.close()


# widths 0..3 mod 4: the scalar tail columns x >= 4 * (w >> 2) of k_sum_minmax
@pytest.mark.parametrize("w", [12, 13, 14, 15, 7])
@pytest.mark.parametrize("c", [1, 3])
def test_stretch_with_the_extremes_in_the_tail_columns_and_last_row(w, c):
    h = 9
    stretch_case(w, h, c, 1, 0, (h - 1, w - 1, c - 1), (0, 0, 0))              # last pixel of the last channel / first
    stretch_case(w, h, c, 1, 0, (0, 0, 0), (h - 1, w - 1, c - 1))
    for x in range(4 * (w >> 2), w):                                          # every tail column, in the last row
        stretch_case(w, h, c, 1, 0, (h - 1, x, c - 1), (h - 2, x, 0))
    stretch_case(w, h, c, 1, 0, (h - 1, 4 * (w >> 2) - 1, c - 1), (2, 3, 0))    # last vector column


def test_stretch_with_more_rows_than_ctas():
    """1 lane: 1185 CTAs share channels * rows = 1203 rows; the extremes in rows that a CTA reaches in its second turn"""
    stretch_case(9, 401, 3, 1, 0, (400, 8, 2), (399, 0, 2))


@pytest.mark.skipif(EMU, reason="70 lanes are too slow for the CPU emulation")
def test_stretch_last_lane_of_70():
    """70 lanes: 17 CTAs a lane share 144 rows"""
    stretch_case(65, 48, 3, 70, 69, (47, 64, 2), (46, 63, 2))


def test_stretch_last_lane_of_3():
    stretch_case(65, 48, 3, 3, 2, (47, 64, 2), (46, 63, 2))
