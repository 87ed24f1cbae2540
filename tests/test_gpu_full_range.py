"""Full-range colour content through the kernels: the corners and edges of the colour cube, shadows, highlights,
saturated and high-frequency content, and outputs that clip at 0 and 255.

The other parity tests feed mid-tone content (lvm_b200.synth.synth_frame, about [42, 214] with correlated channels),
which reaches only the middle LUT cells, never the dark-end sRGB spline and never a clipped output.  Here:
  a. the ingest's Lab (read back through the read-only "lab16" state) is bit-exact with cv2 for every 24-bit colour,
     in every ingest kernel and load path;
  b. the egress pixel stage (a Laplace lane's first frame adds exactly +-0 motion) is within 2e-5 of cv2's Lab2BGR for
     every colour, and its u8 output within 1 LSB, only next to a rounding tie;
  c. egress under teacher-forced extreme motion (Lab far outside its range, outputs clipped) matches the oracle;
  d. every mode runs full-range content kinds against the compiled reference (the oracle if oracle/_ref is absent),
     and clips and multi-lane handles reproduce frame calls bit for bit on that content.

On the CUDA emulation (MC_EMU=1) the exhaustive cases use the lattice-edge colours E^3 instead of all 2^24 colours."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from oracle import livim_oracle as O
from oracle import livim_ref
from common import make_cfgs, planar, u8_diff

pytestmark = pytest.mark.gpu
R = livim_ref.load()
EMU = os.environ.get("MC_EMU") == "1"
F32 = np.float32

# colours next to the LUT lattice (cells are 8.0 u8 steps wide: cell t starts at u8 ~7.94 t), the dark-end spline limit
# and the top of the cube
EDGE = [0, 1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 127, 128, 247, 248, 254, 255]


# ---- content ---------------------------------------------------------------------------------------------------------

def colour_set(edge):
    """(N, 3) u8 BGR.  Every 24-bit colour, pixel i = (b, g, r) = (i >> 16, (i >> 8) & 255, i & 255); with `edge`
    the lattice-edge colours E^3 in the same order."""
    if edge:
        v = np.array(EDGE, np.uint8)
        b, g, r = np.meshgrid(v, v, v, indexing="ij")
        return np.stack([b.ravel(), g.ravel(), r.ravel()], -1)
    i = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8)


_FRAMES = {}


def colour_frame(aligned, edge):
    """Every colour of colour_set(edge) once, as a frame.  aligned: 4096 x 4096 (72 x 81 for E^3), rows of 3w bytes
    4-byte aligned, so the vector load paths run.  Otherwise 4097 x 4097 (77 x 77): rows are not 4-byte aligned, so
    the scalar load paths and the strip tails run; the extra pixels come from a seeded permutation of the colours."""
    key = (aligned, edge)
    if key not in _FRAMES:
        px = colour_set(edge)
        n = len(px)
        w, h = ((72, 81) if edge else (4096, 4096)) if aligned else ((77, 77) if edge else (4097, 4097))
        extra = px[np.random.default_rng(7).permutation(n)[:w * h - n]]
        _FRAMES[key] = np.ascontiguousarray(np.concatenate([px, extra]).reshape(h, w, 3))
    return _FRAMES[key]


def ref_lab(frame):
    return cv2.cvtColor(frame.astype(F32) * F32(1 / 255.0), cv2.COLOR_BGR2Lab)


def decode_lab16(tap):
    """[3][h][w] raw fixed-point Lab (L*2^14/100, (a+128)*64, (b+128)*64) -> h x w x 3 float Lab, as the kernels decode it."""
    return np.stack([tap[0] * F32(100.0 / 16384.0), tap[1] * F32(1 / 64.0) + F32(-128.0), tap[2] * F32(1 / 64.0) + F32(-128.0)], -1)


def lut_cell(v):
    """LUT cell (0 .. 32) that a u8 sample falls in (mc_math.cuh lab_q_of_u8)."""
    return ((v.astype(np.int32) * 16448 + 128) >> 13) >> 4


KINDS = ["blocks", "checker", "shadows", "highlights", "corners", "noise"]


def _corner_palette():
    c = np.array([[b, g, r] for b in (0, 255) for g in (0, 255) for r in (0, 255)], np.int32)
    ramp = np.arange(256)
    edges = []
    for i in range(8):
        for j in range(i + 1, 8):
            if np.count_nonzero(c[i] != c[j]) == 1:   # the 12 edges of the cube
                k = int(np.flatnonzero(c[i] != c[j])[0])
                e = np.repeat(c[i][None], 256, 0)
                e[:, k] = ramp
                edges.append(e)
    return np.concatenate([np.repeat(c, 16, 0)] + edges).astype(np.uint8)


def content(kind, t, w, h, seed=0):
    """Frame t of a seeded full-range content kind (h x w x 3 u8)."""
    y, x = np.mgrid[0:h, 0:w]
    base = np.random.default_rng(seed)
    if kind == "blocks":      # per-channel 0/255 blocks of different sizes, moving a pixel per frame
        return np.stack([((((x + t) // s) + (y // s) + c) % 2) * 255 for c, s in enumerate((3, 5, 8))], -1).astype(np.uint8)
    if kind == "checker":     # 1-px 0/255 checkerboard, a 4-px inverted bar moving 3 px per frame
        f = ((x + y) % 2) * 255
        bar = (x - 3 * t) % max(w, 1) < 4
        return np.repeat(np.where(bar, 255 - f, f)[..., None], 3, -1).astype(np.uint8)
    if kind in ("shadows", "highlights"):   # 0..10 / 245..255, per channel, cycling per frame
        v = (base.integers(0, 11, (h, w, 3)) + t) % 11
        return (v if kind == "shadows" else 245 + v).astype(np.uint8)
    if kind == "corners":     # the 8 corners of the RGB cube and ramps along its 12 edges, shifted per frame
        pal = _corner_palette()
        idx = (base.permutation(h * w) + 37 * t) % len(pal)
        return pal[idx].reshape(h, w, 3)
    if kind == "noise":       # uniform, fresh every frame
        return np.random.default_rng(seed * 1000 + t).integers(0, 256, (h, w, 3), dtype=np.uint8)
    raise ValueError(kind)


def assert_kind_covers(kind, frames):
    """Each kind exists for a property of its content; check it holds."""
    a = np.stack(frames)
    cells = np.unique(lut_cell(a))
    if kind in ("blocks", "checker", "corners", "noise"):
        assert cells[0] == 0 and cells[-1] == 32, (kind, cells)        # both ends of the LUT lattice
    if kind == "corners":
        assert len(np.unique(a.reshape(-1, 3), axis=0)) >= 64          # corners and edge ramps
    if kind == "shadows":
        assert a.max() <= 10 and cells.tolist() == [0, 1]               # linear values below the spline limit
        assert (ref_lab(a[0])[..., 0] <= 8).mean() > 0.5                 # Lab L <= 8: the linear branch of Lab2BGR
    if kind == "highlights":
        assert a.min() >= 245 and cells[-1] == 32
    if kind != "noise" and len(frames) > 1:
        assert not np.array_equal(frames[0], frames[1]), kind            # temporal variation


# ---- a. exhaustive ingest ------------------------------------------------------------------------------------------

INGEST = {   # name: (mode, levels, options, lanes)
    "laplace6 ingest_warps=1": (O.MODE_LAPLACE, 6, {"ingest_warps": 1}, 1),
    "laplace6 ingest_warps=2": (O.MODE_LAPLACE, 6, {"ingest_warps": 2}, 1),
    "laplace6 ingest_warps=4": (O.MODE_LAPLACE, 6, {"ingest_warps": 4}, 1),
    "faithful_level0": (O.MODE_LAPLACE, 6, {"faithful_level0": 1}, 1),
    "laplace1": (O.MODE_LAPLACE, 1, {}, 1),
    "phase": (O.MODE_PHASE, 4, {}, 1),
    "2 lanes lane_groups=2": (O.MODE_LAPLACE, 6, {"lane_groups": 2}, 2),
    "strided rows": (O.MODE_LAPLACE, 6, {}, 1),
}


def run_ingest(name, frame):
    """-> the lab16 planes of every lane after one frame call, and the frames the lanes were given."""
    mode, levels, options, lanes = INGEST[name]
    cfg, _ = make_cfgs(mode, 20, 50.0, 0.4, 3.0, 0, levels)
    proc = L.MagnificationProcessor(0, lanes=lanes)
    for k, v in options.items():
        proc.set_option(k, v)
    h, w = frame.shape[:2]
    if lanes == 2:   # lane 1: a seeded permutation of the colours
        perm = np.random.default_rng(11).permutation(h * w)
        frames = np.stack([frame, frame.reshape(-1, 3)[perm].reshape(h, w, 3)])
        produced, _ = proc.process_image(frames, cfg)
    elif name == "strided rows":   # cv::Mat rows with padding, through the C ABI
        in_step = 3 * w + 5
        src = np.full((h, in_step), 0xAB, np.uint8)
        src[:, :3 * w] = frame.reshape(h, 3 * w)
        frames = frame[None]
        out = np.empty((h, w, 3), np.uint8)
        prod = C.c_int(0)
        p = L.processor._to_mc(cfg)
        assert capi.lib().mc_process(proc._h, src.ctypes.data, w, h, 3, in_step, C.byref(p), out.ctypes.data, 3 * w, C.byref(prod)) == 0
        produced = bool(prod.value)
    else:
        frames = frame[None]
        produced, _ = proc.process_image(frame, cfg)
    assert produced == (mode == O.MODE_LAPLACE)   # a Phase first frame passes through
    tap = proc.get_state("lab16", 0)
    assert tap is not None and tap.shape == (lanes, 3, h, w)
    proc.close()
    return tap, frames


def check_ingest(name, aligned, edge):
    frame = colour_frame(aligned, edge)
    tap, frames = run_ingest(name, frame)
    for lane in range(len(frames)):
        got, ref = decode_lab16(tap[lane]), ref_lab(frames[lane])
        bad = np.argwhere(np.any(got != ref, -1))
        assert len(bad) == 0, (name, lane, len(bad), [(frames[lane][tuple(i)].tolist(), got[tuple(i)].tolist(), ref[tuple(i)].tolist())
                                                    for i in bad[:4]])


@pytest.mark.parametrize("aligned", [True, False], ids=["4096x4096", "4097x4097"])
@pytest.mark.parametrize("name", list(INGEST))
def test_ingest_lab_is_bit_exact_for_every_colour(name, aligned):
    check_ingest(name, aligned, EMU)


def check_lab16_lifecycle(mode):
    """"lab16" exists only after a frame call on 3-channel input, never holds stale planes, and is read-only."""
    cfg, _ = make_cfgs(mode, 20, 50.0, 0.4, 3.0, 0, 3)
    w, h = 67, 35
    f = [content("noise", t, w, h) for t in range(3)]
    proc = L.MagnificationProcessor(0, lanes=2)
    assert proc.get_state("lab16") is None                                  # before any frame
    proc.process_image(np.stack([f[0], f[1]]), cfg)
    tap = proc.get_state("lab16")
    for lane, fr in enumerate((f[0], f[1])):
        assert np.array_equal(decode_lab16(tap[lane]), ref_lab(fr))
    assert proc.state_dims("lab16", 1) == (0, 0, 0)                          # level 0 only
    with pytest.raises(L.MagcoreError) as e:
        proc.set_state("lab16", 0, tap)
    assert e.value.status == capi.MC_ERR_INVALID                            # read-only
    proc.hold_lane(1)                                                       # a held lane keeps its planes
    proc.process_image(np.stack([f[2], f[2]]), cfg)
    tap = proc.get_state("lab16")
    assert np.array_equal(decode_lab16(tap[0]), ref_lab(f[2])) and np.array_equal(decode_lab16(tap[1]), ref_lab(f[1]))
    proc.hold_lane(1, False)
    proc.process_clip(np.stack([np.stack([f[0], f[1]])] * 2), cfg)
    assert proc.get_state("lab16") is None                                  # after a clip call
    proc.process_image(np.stack([f[0], f[1]]), cfg)
    assert proc.get_state("lab16") is not None
    proc.reset()
    assert proc.get_state("lab16") is None                                  # after reset
    proc.process_image(np.stack([f[0][..., 0].copy(), f[1][..., 0].copy()]), cfg)
    assert proc.get_state("lab16") is None                                  # gray input has no Lab planes
    proc.close()


@pytest.mark.parametrize("mode", [O.MODE_LAPLACE, O.MODE_PHASE], ids=["laplace", "phase"])
def test_lab16_state_lifecycle(mode):
    check_lab16_lifecycle(mode)


# ---- b. exhaustive egress pixel stage ------------------------------------------------------------------------------

FLOAT_TWIN_TOL = 2e-5   # tests/test_host.py: what the host twin of the conversion meets against cv2


def check_egress_pixel_stage(aligned, edge, against_ref):
    """First frame of a Laplace lane: output = Lab2BGR(Lab16 of the input), no motion.  Returns (max float error,
    number of 1-LSB u8 differences)."""
    frame = colour_frame(aligned, edge)
    h, w = frame.shape[:2]
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 0, 6)
    res = {}
    for strip in (20, 0):
        proc = L.MagnificationProcessor(0)
        proc.set_option("keep_float_output", 1)
        proc.set_option("egress_strip", strip)
        produced, out = proc.process_image(frame, cfg)
        assert produced
        res[strip] = (out, proc.float_output(w, h, 3)[0], proc.get_state("lab16")[0])
        proc.close()
    out, fo, tap = res[20]
    assert np.array_equal(out, res[0][0]) and np.array_equal(fo, res[0][1])   # strip and tile egress: bit-identical
    lab = decode_lab16(tap)
    ref_f = cv2.cvtColor(lab, cv2.COLOR_Lab2BGR)
    err = float(np.abs(fo - ref_f).max())
    assert err < FLOAT_TWIN_TOL, err
    ref_u8 = O._f32_to_u8(ref_f, 255.0, 1.0 / 255.0)
    d = u8_diff(out, ref_u8)
    assert int(d.max()) <= 1
    # a float error of at most 2e-5 can move the rounding only when the reference lies that close to a tie
    v = ref_f[d == 1].astype(np.float64) * 255.0 + 1.0 / 255.0
    tie = np.abs(v - np.floor(v) - 0.5)
    assert bool(np.all(tie <= FLOAT_TWIN_TOL * 255.0)), float(tie.max())
    if against_ref and R is not None:
        rout = R.Processor().process(frame, livim_ref.to_ref_config(R, ocfg))[1]
        assert int(u8_diff(out, rout).max()) <= 1
    return err, int((d == 1).sum())


@pytest.mark.parametrize("aligned", [True, False], ids=["4096x4096", "4097x4097"])
def test_egress_pixel_stage_for_every_colour(aligned):
    err, n1 = check_egress_pixel_stage(aligned, EMU, against_ref=aligned)
    print(f"egress pixel stage {'aligned' if aligned else 'unaligned'}: max float error {err:.3g}, 1-LSB pixels {n1}")


# ---- c. egress under extreme motion (teacher-forced) ---------------------------------------------------------------

def extreme_frame(w, h, c, seed):
    """Noise with a band of shadows (L <= 8) and one of highlights."""
    f = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    f[: h // 4] //= 24
    f[h // 4: h // 2] = 235 + f[h // 4: h // 2] // 13
    return f if c == 3 else np.ascontiguousarray(f[..., 1])


def check_extreme_motion(c, levels, strip, w=333, h=251):
    cfg, ocfg = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 100, levels)
    proc, oproc = L.MagnificationProcessor(0), O.MagnificationProcessor()
    proc.set_option("keep_float_output", 1)
    proc.set_option("egress_strip", strip)
    proc.process_image(extreme_frame(w, h, c, 0), cfg)
    oproc.process(extreme_frame(w, h, c, 0), ocfg)
    rng = np.random.default_rng(100 + levels)
    scale = 12.0 if c == 3 else 0.12   # Lab units / [0, 1] units; every live band has gain 20 at this size
    for lvl in range(1, levels):   # the live bands: the only state the production path keeps
        shape = oproc.motion.lowpassHi[lvl].shape
        blocks = np.kron(rng.uniform(-1, 1, (shape[0] // 2 + 1, shape[1] // 2 + 1) + shape[2:]),
                         np.ones((2, 2) + (1,) * (len(shape) - 2)))[:shape[0], :shape[1]]
        hi = (oproc.motion.lowpassHi[lvl] + scale * blocks).astype(F32)
        lo = (oproc.motion.lowpassLo[lvl] - scale * blocks).astype(F32)
        oproc.motion.lowpassHi[lvl], oproc.motion.lowpassLo[lvl] = hi.copy(), lo.copy()
        proc.set_state("lowpassHi", lvl, planar(hi)[None])
        proc.set_state("lowpassLo", lvl, planar(lo)[None])
    f = extreme_frame(w, h, c, 1)
    dbg = {}
    produced, out = proc.process_image(f, cfg)
    oprod, oout = oproc.process(f, ocfg, dbg)
    assert produced and oprod
    ref_f = dbg["output_bgr_f32"] if c == 3 else dbg["output_f32"]
    got_f = proc.float_output(w, h, c)[0]
    if c == 1:
        got_f = got_f[..., 0]
    # coverage: what this test exists for
    assert (oout == 0).mean() >= 0.05 and (oout == 255).mean() >= 0.05, ((oout == 0).mean(), (oout == 255).mean())
    assert (ref_f < 21 / 255).mean() >= 0.05
    if c == 3:
        lab = dbg["output_f32"]
        assert lab[..., 0].min() < -20 and lab[..., 0].max() > 120, (lab[..., 0].min(), lab[..., 0].max())
        assert np.abs(lab[..., 1]).max() > 128 and np.abs(lab[..., 2]).max() > 128
        assert (dbg["input_f32"][..., 0] <= 8).any() and ((lab[..., 0] <= 8) & (lab[..., 0] >= 0)).any()
    err = float(np.abs(got_f - ref_f).max())
    assert err < 1e-4, err
    assert int(u8_diff(out, oout).max()) <= 1


@pytest.mark.parametrize("strip", [20, 0])
@pytest.mark.parametrize("levels", [2, 3, 5], ids=["L2-no-c2", "L3-c2-from-state", "L5-collapse"])
@pytest.mark.parametrize("c", [3, 1])
def test_egress_under_extreme_motion(c, levels, strip):
    check_extreme_motion(c, levels, strip)


# ---- d. full-range parity against the compiled reference ----------------------------------------------------------

MODES = {   # name: (mode, ui, fps, frames, channels)
    "laplace c3 a20 ch0 L2": (O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 2), 30.0, 5, 3),
    "laplace c3 a200 ch100 L4": (O.MODE_LAPLACE, (200, 50.0, 0.4, 3.0, 100, 4), 30.0, 5, 3),
    "laplace c3 a20 ch100 L9": (O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 100, 9), 30.0, 5, 3),
    "laplace c1 a20 L2": (O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 2), 30.0, 5, 1),
    "laplace c1 a200 L4": (O.MODE_LAPLACE, (200, 50.0, 0.4, 3.0, 100, 4), 30.0, 5, 1),
    "laplace c1 a20 L9": (O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 100, 9), 30.0, 5, 1),
    "phase defaults": (O.MODE_PHASE, (20, 50.0, 1.0, 2.5, 0, 4), 30.0, 5, 3),
    "phase a150": (O.MODE_PHASE, (150, 50.0, 1.0, 2.5, 0, 4), 30.0, 5, 3),
    "color 8fps": (O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 2), 8.0, 20, 3),
}


def kind_frames(kind, w, h, n, c):
    fr = [content(kind, t, w, h) for t in range(n)]
    assert_kind_covers(kind, fr)
    return fr if c == 3 else [np.ascontiguousarray(cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)) for f in fr]


def check_parity(mname, kind, w, h, n=None):
    mode, ui, fps, nf, c = MODES[mname]
    frames = kind_frames(kind, w, h, n or nf, c)
    cfg, ocfg = make_cfgs(mode, *ui, fps)
    proc = L.MagnificationProcessor(0)
    use_ref = R is not None
    ref, rcfg = (R.Processor(), livim_ref.to_ref_config(R, ocfg)) if use_ref else (O.MagnificationProcessor(), ocfg)
    if mode == O.MODE_LAPLACE and not use_ref:
        proc.set_option("keep_float_output", 1)
    for t, f in enumerate(frames):
        produced, out = proc.process_image(f, cfg)
        dbg = {}
        rprod, rout = ref.process(f, rcfg) if use_ref else ref.process(f, rcfg, dbg)
        assert produced == bool(rprod), (mname, kind, t)
        if not produced:
            continue
        d = u8_diff(out, rout)
        if mode == O.MODE_PHASE:
            assert int(d.max()) <= 3 and float((d == 0).mean()) >= 0.995, (mname, kind, t, int(d.max()), float((d == 0).mean()))
        else:
            assert int(d.max()) <= 1, (mname, kind, t, int(d.max()))
        if mode == O.MODE_LAPLACE and not use_ref:
            got_f = proc.float_output(w, h, c)[0]
            ref_f = dbg["output_bgr_f32"] if c == 3 else dbg["output_f32"][..., None]
            assert float(np.abs(got_f - ref_f).max()) < 1e-4, (mname, kind, t)
    proc.close()


@pytest.mark.parametrize("w,h", [(129, 67), (241, 135), (7, 9)], ids=["129x67", "241x135", "7x9"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mname", list(MODES))
def test_full_range_parity(mname, kind, w, h):
    check_parity(mname, kind, w, h)


@pytest.mark.parametrize("mname,kind", [("laplace c3 a200 ch100 L4", "blocks"), ("phase a150", "checker"), ("color 8fps", "noise")])
def test_full_range_parity_1080p(mname, kind):
    check_parity(mname, kind, 1920, 1080, n=MODES[mname][3] if MODES[mname][0] == O.MODE_COLOR else 3)


def check_clip_equals_frames(mname, kind, w, h, T=6):
    mode, ui, fps, _, c = MODES[mname]
    frames = np.stack(kind_frames(kind, w, h, 2 * T, c))
    cfg, _ = make_cfgs(mode, *ui, fps)
    a, b = L.MagnificationProcessor(0), L.MagnificationProcessor(0)
    for k in range(2):   # a fresh clip, then a continuing one
        seg = frames[k * T:(k + 1) * T]
        flags, outs = a.process_clip(seg, cfg)
        for t in range(T):
            produced, out = b.process_image(seg[t], cfg)
            assert bool(flags[t, 0]) == produced and np.array_equal(outs[t], out), (mname, kind, k, t)
    a.close()
    b.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mname", ["laplace c3 a200 ch100 L4", "laplace c1 a200 L4", "phase a150"])
def test_clip_equals_frame_calls_on_full_range_content(mname, kind):
    check_clip_equals_frames(mname, kind, 129, 67)


def check_lanes_equal_single(mname, kinds, w, h, n=4):
    mode, ui, fps, _, c = MODES[mname]
    per = [kind_frames(k, w, h, n, c) for k in kinds]
    cfg, _ = make_cfgs(mode, *ui, fps)
    multi = L.MagnificationProcessor(0, lanes=len(kinds))
    singles = [L.MagnificationProcessor(0) for _ in kinds]
    for t in range(n):
        _, mout = multi.process_image(np.stack([p[t] for p in per]), cfg)
        for i, s in enumerate(singles):
            _, out = s.process_image(per[i][t], cfg)
            assert np.array_equal(mout[i], out), (mname, kinds[i], t)
    for p in [multi] + singles:
        p.close()


@pytest.mark.parametrize("mname", ["laplace c3 a200 ch100 L4", "laplace c1 a20 L2", "phase a150", "color 8fps"])
def test_lanes_with_different_kinds_equal_single_lane_handles(mname):
    check_lanes_equal_single(mname, ["blocks", "shadows", "highlights", "noise"], 129, 67,
                             n=10 if MODES[mname][0] == O.MODE_COLOR else 4)
