"""Moving a lane's temporal state (mc_save_lane / mc_load_lane): lane k of handle A is saved, the blob is loaded into lane
j of handle B, and from then on lane j, fed lane k's frames with lane k's parameters, must give bit for bit what lane k
gives: outputs, produced flags, mc_lane_produced and the temporal state.  B's other lanes must equal a twin of B without
the load, and A a twin of A without the save.  The continuation runs through frame calls, clips, pinned and pageable
submits, chain submits of BGR, NV12 and YUYV frames and compose submits, in all three modes."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from test_gpu_lanes import COLOR_UI, LAPLACE_UI, PHASE_UI, SENTINEL, state_names
from test_gpu_lane_params import cfg_of, effective, mag

pytestmark = pytest.mark.gpu

# every continuation entry point, one call each: (entry, frames per call)
ENTRIES = [("frame", 1), ("clip", 3), ("submit", 1), ("submit_pinned", 1), ("chain", 1), ("nv12", 1), ("yuyv", 1),
           ("compose", 2), ("frame", 1)]


def frame_of(stream, t, w, h, c):
    return synth_frame(t, w, h, c, seed=101 * stream + 7)


class Pinned:
    """Page-locked host arrays (mc_host_alloc), freed with the object."""

    def __init__(self):
        self.ptrs = []

    def array(self, shape):
        lib = capi.lib()
        n = int(np.prod(shape))
        p = lib.mc_host_alloc(n)
        assert p
        self.ptrs.append(p)
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(p)).reshape(shape)

    def __del__(self):
        for p in self.ptrs:
            capi.lib().mc_host_free(p)


class Handle:
    """A chain handle with one source stream per lane (stream ids index frame_of) and per-lane overrides."""

    def __init__(self, lanes, streams, options=(), device=0):
        self.chain = L.ProcessingChainB200(device, lanes)
        self.m = self.chain.magnifier
        self.lanes = lanes
        self.streams = list(streams)
        for key, v in options:
            self.m.set_option(key, v)

    def frames(self, t0, n, w, h, c):
        return np.stack([np.stack([frame_of(s, t0 + t, w, h, c) for s in self.streams]) for t in range(n)])

    def feed(self, entry, t0, n, w, h, c, params, pinned):
        """One call of `entry` over n frames from t0 -> (flags bool[n, lanes], per-lane outputs [n, lanes, ...])."""
        cfg = cfg_of(params)
        f = self.frames(t0, n, w, h, c)
        lanes, m, ch = self.lanes, self.m, self.chain
        if entry == "frame":
            out = np.full_like(f[0], SENTINEL)
            m.process_host(f[0].ctypes.data, w, h, c, w * c, cfg, out.ctypes.data, w * c)
            return m.lane_produced()[None], out[None]
        if entry == "clip":
            out = np.full_like(f, SENTINEL)
            flags = np.zeros((n, lanes), np.uint8)
            m._check(m._lib.mc_process_clip(m._h, f.ctypes.data, n, w, h, c, w * c, C.byref(L.processor._to_mc(cfg)),
                                            out.ctypes.data, w * c, flags.ctypes.data_as(C.POINTER(C.c_uint8))))
            assert np.array_equal(flags[-1].astype(bool), m.lane_produced())
            return flags.astype(bool), out
        if entry in ("submit", "submit_pinned"):
            src = f[0] if entry == "submit" else pinned.array(f[0].shape)
            src[...] = f[0]
            out = np.full_like(f[0], SENTINEL) if entry == "submit" else pinned.array(f[0].shape)
            out[...] = SENTINEL
            m.submit(src.ctypes.data, w, h, c, w * c, cfg, out.ctypes.data, w * c)
            m.collect()
            return m.lane_produced()[None], out.copy()[None]
        assert c == 3
        out = np.full((lanes, h, w, 3), SENTINEL, np.uint8)
        if entry == "chain":
            ch.submit(f[0].ctypes.data, w, h, 3, w * 3, cfg, out.ctypes.data, w * 3)
        elif entry == "nv12":   # any bytes are an NV12 frame: luma from B, chroma from G of the even rows
            nv = np.ascontiguousarray(np.concatenate([f[0][:, :, :, 0], f[0][:, ::2, :, 1]], axis=1))
            ch.submit_nv12(capi.McNv12(nv.ctypes.data, nv.ctypes.data + w * h, w, w * h * 3 // 2), w, h, cfg, out.ctypes.data, w * 3)
        elif entry == "yuyv":
            yv = np.ascontiguousarray(f[0][:, :, :, :2]).reshape(lanes, h, 2 * w)
            ch.submit_yuv422(capi.McYuv422(yv.ctypes.data, 2 * w, 2 * w * h, capi.MC_YUV422_YUYV), w, h, cfg, out.ctypes.data, w * 3)
        elif entry == "compose":
            cw, chh = w & ~1, h & ~1
            out = np.full((n, lanes, chh, cw, 3), SENTINEL, np.uint8)
            canvas = capi.McCanvas(capi.MC_CANVAS_BGR, out.ctypes.data, None, cw * 3, cw * chh * 3)
            _, flags = ch.compose_submit(f.ctypes.data, n, w, h, 3, w * 3, cfg, capi.MC_SPLIT_NONE, canvas)
            ch.collect()
            return flags.astype(bool), out
        else:
            raise ValueError(entry)
        ch.collect()
        return m.lane_produced()[None], out[None]


def lane_states(hd, mode):
    """name -> f32 [lanes, ...] of every temporal state plane set (Color: the window columns every lane has)."""
    if mode == O.MODE_COLOR:
        names = [("window", l) for l in range(128) if hd.m.state_dims("window", l)[0]]
    else:
        names = state_names(hd.m, mode)
    return {nl: hd.m.get_state(*nl) for nl in names}


def compare(a, b, la, lb, what):
    """Lane la of handle a's flags / outputs / states against lane lb of b."""
    (fa, oa, sa), (fb, ob, sb) = a, b
    assert np.array_equal(fa[:, la], fb[:, lb]), (what, "flags")
    assert np.array_equal(oa[:, la], ob[:, lb]), (what, "out")
    common = set(sa) & set(sb)
    assert common or not (sa or sb), (what, "no common state")
    for nl in common:
        assert np.array_equal(sa[nl][la], sb[nl][lb], equal_nan=True), (what, nl)


@dataclasses.dataclass
class Move:
    mode: int
    ui: tuple
    w: int
    h: int
    c: int = 3
    a_lanes: int = 3
    k: int = 1
    b_lanes: int = 2
    j: int = 0
    before: int = 4            # frames A runs before the save
    b_before: int = 3          # frames B runs before the load (0: a new handle)
    options: tuple = ()
    a_params: object = None    # A's call params before the save (default: mag(mode, ui))
    params: object = None      # every handle's call params after the move (default: a_params)
    a_over: tuple = ()         # A's per-lane overrides (MagnificationParams or None), padded with None
    b_over: tuple = ()
    same_handle: bool = False  # B is A (and B's twin A's)
    entries: tuple = tuple(ENTRIES)
    hooks: dict = dataclasses.field(default_factory=dict)   # call index -> fn(A, A2, B, B2) before that call
    prepare: object = None     # fn(A, A2, B, B2) after the runs before the move, before the save
    b_device: int = 0


def check_move(mv: Move):
    w, h, c = mv.w, mv.h, mv.c
    a_params = mv.a_params or mag(mv.mode, mv.ui)
    params = mv.params or a_params
    a_over = list(mv.a_over) + [None] * (mv.a_lanes - len(mv.a_over))
    b_over = list(mv.b_over) + [None] * (mv.b_lanes - len(mv.b_over))
    A, A2 = (Handle(mv.a_lanes, range(mv.a_lanes), mv.options) for _ in range(2))
    for hd in (A, A2):
        for l, o in enumerate(a_over):
            if o is not None:
                hd.m.set_lane_params(l, o)
    if mv.same_handle:
        B, B2 = A, A2
    else:
        B, B2 = (Handle(mv.b_lanes, [100 + i for i in range(mv.b_lanes)], mv.options, mv.b_device) for _ in range(2))
        for hd in (B, B2):
            for l, o in enumerate(b_over):
                if o is not None:
                    hd.m.set_lane_params(l, o)
    pinned = Pinned()
    for t in range(mv.before):
        ra, ra2 = A.feed("frame", t, 1, w, h, c, a_params, pinned), A2.feed("frame", t, 1, w, h, c, a_params, pinned)
        assert all(np.array_equal(x, y) for x, y in zip(ra, ra2))
    if not mv.same_handle:
        for t in range(mv.b_before):
            B.feed("frame", t, 1, w, h, c, params, pinned)
            B2.feed("frame", t, 1, w, h, c, params, pinned)
    if mv.prepare:
        mv.prepare(A, A2, B, B2)

    blob = A.m.save_lane(mv.k)
    B.m.load_lane(mv.j, blob)
    assert B.m.save_lane(mv.j) == blob   # save -> load -> save: the same bytes
    # the stream moves with its parameters; B's twin keeps lane j as it was
    B.m.set_lane_params(mv.j, a_over[mv.k])
    B.streams[mv.j] = A.streams[mv.k]
    if not mv.same_handle:
        B2.streams[mv.j] = A.streams[mv.k]   # the twin's lane j is not compared

    t = mv.before
    for i, (entry, n) in enumerate(mv.entries):
        if i in mv.hooks:
            mv.hooks[i](A, A2, B, B2)
        if c == 1 and entry in ("chain", "nv12", "yuyv", "compose"):
            continue
        rb = B.feed(entry, t, n, w, h, c, params, pinned) + (None,)
        rb2 = B2.feed(entry, t, n, w, h, c, params, pinned) + (None,)
        ra = rb if mv.same_handle else A.feed(entry, t, n, w, h, c, params, pinned) + (None,)
        ra2 = rb2 if mv.same_handle else A2.feed(entry, t, n, w, h, c, params, pinned) + (None,)
        sa, sa2, sb, sb2 = (lane_states(x, mv.mode) for x in (A, A2, B, B2))
        ra, ra2, rb, rb2 = ((r[0], r[1], s) for r, s in ((ra, sa), (ra2, sa2), (rb, sb), (rb2, sb2)))
        what = (entry, t)
        compare(rb, ra2, mv.j, mv.k, what + ("moved lane",))
        for l in range(mv.b_lanes if not mv.same_handle else mv.a_lanes):
            if l != mv.j:
                compare(rb, rb2, l, l, what + ("other lane", l))
        if not mv.same_handle:
            for l in range(mv.a_lanes):
                compare(ra, ra2, l, l, what + ("source", l))
        t += n
    return A, B


# ---------------------------------------------------------------------------------------------------------------------
# checks shared with the emulation suite (tests/test_emu_lane_state.py)
# ---------------------------------------------------------------------------------------------------------------------
def laplace_over(k, chroma=None, coLow=None):
    base = mag(O.MODE_LAPLACE, LAPLACE_UI)
    ui = ((5 + 7 * k) % 41 + 1, 20.0 + (9 * k) % 61, 0.2 + 0.05 * k, 1.5 + 0.25 * k, [0, 50, 20][k % 3] if chroma is None else chroma, 4)
    o = effective(base, mag(O.MODE_LAPLACE, ui, [25.0, 30.0, 60.0][k % 3]))
    return o if coLow is None else dataclasses.replace(o, coLow=coLow)


def check_laplace(w, h, entries=tuple(ENTRIES)):
    """Colour at chroma 0 and 50, gray, per-lane params, faithful_level0 and two lane groups."""
    for chroma in (0, 50):
        p = dataclasses.replace(mag(O.MODE_LAPLACE, LAPLACE_UI), chromAttenuation=chroma / 100.0)
        check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, a_params=p, entries=entries))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, c=1, entries=entries))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, a_over=(laplace_over(0), laplace_over(1), None),
                    b_over=(laplace_over(2), laplace_over(0)), entries=entries))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, options=(("faithful_level0", 1),), entries=entries[:3]))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, a_lanes=4, k=3, b_lanes=4, j=1, options=(("lane_groups", 2),),
                    entries=entries[:4]))


def check_laplace_unbounded(w, h):
    """A source whose state is not bounded by its bands into a bounded handle at chroma 0: the destination must stop
    synthesising L alone, whatever the moved lane's cutoffs.  With cutoffs in [0, 1] only the blob says so: its state of
    +-3e38 makes the a / b motion overflow, which L-only synthesis would drop.  With coLow > 1 (state +-1e7) the lane's
    own cutoffs say so too."""
    p = dataclasses.replace(mag(O.MODE_LAPLACE, LAPLACE_UI), chromAttenuation=0.0)

    def blow_up(v):
        def f(A, A2, B, B2):
            rng = np.random.default_rng(5)
            for name, lv in state_names(A.m, O.MODE_LAPLACE):
                s = A.m.get_state(name, lv)
                s[1] = rng.choice([-v, v], size=s[1].shape).astype(np.float32)
                A.m.set_state(name, lv, s)
                A2.m.set_state(name, lv, s)
        return f

    entries = (("frame", 1), ("clip", 2), ("frame", 1))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, a_params=p, a_over=(None, laplace_over(1, chroma=0)),
                    prepare=blow_up(3e38), entries=entries))
    check_move(Move(O.MODE_LAPLACE, LAPLACE_UI, w, h, a_params=p, a_over=(None, laplace_over(1, chroma=0, coLow=1.5)),
                    prepare=blow_up(1e7), entries=entries))


def check_phase(w, h, entries=tuple(ENTRIES)):
    """The source lane designed at 25 fps, the destination's lanes at 30; a cutoff change right after the load
    re-designs at 25 fps."""
    p25 = dataclasses.replace(mag(O.MODE_PHASE, PHASE_UI), framerate=25.0)
    p30 = dataclasses.replace(p25, framerate=30.0)
    check_move(Move(O.MODE_PHASE, PHASE_UI, w, h, a_params=p25, params=p30, entries=entries))
    moved = dataclasses.replace(p30, coLow=0.6, coHigh=2.5)

    def cutoffs(A, A2, B, B2):
        for hd, l in ((A, 1), (A2, 1), (B, 0)):
            hd.m.set_lane_params(l, moved)

    check_move(Move(O.MODE_PHASE, PHASE_UI, w, h, a_params=p25, params=p30, hooks={0: cutoffs},
                    entries=(("frame", 1), ("frame", 1), ("clip", 3), ("frame", 1))))


def check_color(w, h, n_tail=15):
    """Windows partly filled (count < mod), full and wrapped (head != 0), and a destination ring smaller than the
    lane's window (15 fps: 32 slots, into a handle at 8 fps: 16 slots)."""
    opts = (("color_lane_lifecycle", 1),)
    base = mag(O.MODE_COLOR, COLOR_UI)
    f8, f15 = (dataclasses.replace(base, framerate=f) for f in (8.0, 15.0))
    entries = (("frame", 1), ("clip", 3), ("submit", 1), ("chain", 1), ("compose", 2), ("nv12", 1)) + (("frame", 1),) * n_tail
    check_move(Move(O.MODE_COLOR, COLOR_UI, w, h, before=5, options=opts, a_params=f8, entries=entries))     # count 5 < 16
    check_move(Move(O.MODE_COLOR, COLOR_UI, w, h, before=21, options=opts, a_params=f8, entries=entries))    # wrapped
    check_move(Move(O.MODE_COLOR, COLOR_UI, w, h, before=37, b_before=20, options=opts, a_params=f15, params=f8,
                    a_over=(None, f15), entries=entries))                                                 # ring 16 < 32
    check_move(Move(O.MODE_COLOR, COLOR_UI, w, h, before=9, b_before=0, a_lanes=1, k=0, b_lanes=1, a_params=f8,
                    entries=entries[:8]))


def check_moves(w, h):
    """Lane -> other lane of the same handle, into a new handle and after mc_reset, into a held lane released later,
    and a lane without state (its blob loads as a restart)."""
    ui = LAPLACE_UI
    check_move(Move(O.MODE_LAPLACE, ui, w, h, same_handle=True, k=0, j=2, entries=ENTRIES[:5]))
    check_move(Move(O.MODE_LAPLACE, ui, w, h, b_before=0, entries=ENTRIES[:5]))
    check_move(Move(O.MODE_PHASE, PHASE_UI, w, h, b_before=0, entries=ENTRIES[:5]))

    def reset(A, A2, B, B2):
        B.m.reset()
        B2.m.reset()

    check_move(Move(O.MODE_LAPLACE, ui, w, h, prepare=reset, entries=ENTRIES[:5]))

    def hold(on):
        def f(A, A2, B, B2):
            for hd, l in ((A, 1), (A2, 1), (B, 0), (B2, 0)):
                hd.m.hold_lane(l, on)
        return f

    check_move(Move(O.MODE_LAPLACE, ui, w, h, prepare=hold(True), hooks={2: hold(False)}, entries=ENTRIES[:6]))
    check_move(Move(O.MODE_PHASE, PHASE_UI, w, h, prepare=hold(True), hooks={2: hold(False)}, entries=ENTRIES[:6]))

    def restart(A, A2, B, B2):
        A.m.restart_lane(1)
        A2.m.restart_lane(1)

    for mode, ui2 in ((O.MODE_LAPLACE, ui), (O.MODE_PHASE, PHASE_UI)):
        check_move(Move(mode, ui2, w, h, prepare=restart, entries=ENTRIES[:3]))


def check_errors(w, h):
    """Every refused save or load leaves both handles equal to twins that never saw it."""
    lib = capi.lib()
    p = mag(O.MODE_LAPLACE, LAPLACE_UI)
    pinned = Pinned()
    A, A2, B, B2 = Handle(2, (0, 1)), Handle(2, (0, 1)), Handle(2, (5, 6)), Handle(2, (5, 6))
    for t in range(3):
        for hd in (A, A2, B, B2):
            hd.feed("frame", t, 1, w, h, 3, p, pinned)
    blob = A.m.save_lane(1)
    n = C.c_size_t(0)
    buf = C.create_string_buffer(len(blob))

    def refused(st, status=capi.MC_ERR_INVALID):
        assert st == status, (st, status)

    refused(lib.mc_save_lane(None, 0, None, 0, C.byref(n)))
    refused(lib.mc_save_lane(A.m._h, 0, None, 0, None))
    for lane in (-1, 2):
        refused(lib.mc_save_lane(A.m._h, lane, None, 0, C.byref(n)))
        refused(lib.mc_load_lane(B.m._h, lane, blob, len(blob)))
    refused(lib.mc_save_lane(A.m._h, 1, buf, len(blob) - 1, C.byref(n)))
    refused(lib.mc_load_lane(None, 0, blob, len(blob)))
    refused(lib.mc_load_lane(B.m._h, 0, None, len(blob)))
    refused(lib.mc_load_lane(B.m._h, 0, blob, len(blob) - 1))       # truncated
    refused(lib.mc_load_lane(B.m._h, 0, blob[:100], 100))
    refused(lib.mc_load_lane(B.m._h, 0, b"X" + blob[1:], len(blob)))  # magic
    bad_version = bytearray(blob)
    bad_version[8] += 1
    refused(lib.mc_load_lane(B.m._h, 0, bytes(bad_version), len(blob)))
    # a key that differs: a blob of another size, another mode
    other = Handle(1, (0,))
    other.feed("frame", 0, 1, w + 2, h, 3, p, pinned)
    refused(lib.mc_load_lane(B.m._h, 0, other.m.save_lane(0), len(other.m.save_lane(0))))
    ph = Handle(1, (0,))
    ph.feed("frame", 0, 1, w, h, 3, mag(O.MODE_PHASE, PHASE_UI), pinned)
    refused(lib.mc_load_lane(B.m._h, 0, ph.m.save_lane(0), len(ph.m.save_lane(0))))
    # faithful_level0 that differs from the destination's
    fa = Handle(1, (0,), (("faithful_level0", 1),))
    fa.feed("frame", 0, 1, w, h, 3, p, pinned)
    refused(lib.mc_load_lane(B.m._h, 0, fa.m.save_lane(0), len(fa.m.save_lane(0))))
    # submitted frames in flight
    f = A.frames(3, 1, w, h, 3)[0]
    out = np.empty_like(f)
    for hd in (A, A2):
        hd.m.submit(f.ctypes.data, w, h, 3, w * 3, cfg_of(p), out.ctypes.data, w * 3)
    refused(lib.mc_save_lane(A.m._h, 0, None, 0, C.byref(n)))
    refused(lib.mc_load_lane(A.m._h, 0, blob, len(blob)))
    for hd in (A, A2):
        hd.m.collect()
    # Color without color_lane_lifecycle on a multi-lane handle
    cA, cB, cB2 = Handle(1, (0,)), Handle(2, (5, 6)), Handle(2, (5, 6))
    pc = mag(O.MODE_COLOR, COLOR_UI)
    for t in range(3):
        for hd in (cA, cB, cB2):
            hd.feed("frame", t, 1, w, h, 3, pc, pinned)
    refused(lib.mc_load_lane(cB.m._h, 1, cA.m.save_lane(0), len(cA.m.save_lane(0))), capi.MC_ERR_UNSUPPORTED)
    refused(lib.mc_load_lane(B.m._h, 1, cA.m.save_lane(0), len(cA.m.save_lane(0))))   # a key that differs
    for t in range(4, 8):
        for a, b, pp in ((A, A2, p), (B, B2, p), (cB, cB2, pc)):
            ra, rb = a.feed("frame", t, 1, w, h, 3, pp, pinned), b.feed("frame", t, 1, w, h, 3, pp, pinned)
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]), t
    for a, b in ((A, A2), (B, B2)):
        sa, sb = lane_states(a, O.MODE_LAPLACE), lane_states(b, O.MODE_LAPLACE)
        assert sa.keys() == sb.keys() and all(np.array_equal(sa[x], sb[x]) for x in sa)


def check_blob_sizes(w, h):
    """A blob's size follows from its key: header + the planes the header names; a lane without state saves the header."""
    pinned = Pinned()
    fresh = Handle(2, (0, 1))
    empty = fresh.m.save_lane(0)
    hd = Handle(2, (0, 1))
    hd.feed("frame", 0, 1, w, h, 3, mag(O.MODE_LAPLACE, LAPLACE_UI), pinned)
    full = hd.m.save_lane(1)
    planes = sum(2 * hd.m.get_state("lowpassHi", l)[1].nbytes for l in range(1, 4))
    assert len(full) - len(empty) == planes
    fresh.m.load_lane(1, empty)   # a restart: nothing to run on
    assert fresh.m.save_lane(1) == empty


# ---------------------------------------------------------------------------------------------------------------------
def test_laplace_moves_through_every_entry_point():
    check_laplace(96, 64)


def test_laplace_unbounded_state_turns_luma_only_synthesis_off():
    check_laplace_unbounded(96, 64)


def test_phase_lane_keeps_its_design_framerate():
    check_phase(96, 64)


def test_color_window_keeps_its_ring_layout():
    check_color(96, 64)


def test_moves_between_lanes_handles_resets_holds():
    check_moves(96, 64)


def test_refused_saves_and_loads_change_nothing():
    check_errors(96, 64)


def test_blob_sizes():
    check_blob_sizes(96, 64)


def test_bench_shape_one_lane_of_64_at_1080p():
    """One lane of the bench's 64-lane 1080p Laplace shape into lane 0 of a new 1-lane handle."""
    w, h, lanes, k = 1920, 1080, 64, 37
    p = mag(O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 6))
    cfg = cfg_of(p)
    base = [synth_frame(t, w, h, 3) for t in range(6)]
    frames = [np.stack([np.roll(f, (11 * l, 37 * l), axis=(0, 1)) for l in range(lanes)]) for f in base]
    A, B = L.MagnificationProcessor(0, lanes=lanes), L.MagnificationProcessor(0, lanes=1)

    def run(m, f):
        out = np.full_like(f, SENTINEL)
        m.process_host(f.ctypes.data, w, h, 3, w * 3, cfg, out.ctypes.data, w * 3)
        return m.lane_produced(), out

    for t in range(3):
        run(A, frames[t])
    blob = A.save_lane(k)
    assert abs(len(blob) / 1e6 - 16.6) < 0.1
    B.load_lane(0, blob)
    for t in range(3, 5):
        (fa, oa), (fb, ob) = run(A, frames[t]), run(B, np.ascontiguousarray(frames[t][k:k + 1]))
        assert fa[k] == fb[0] and np.array_equal(oa[k], ob[0]), t
    fa, oa = A.process_clip(frames[5][None], cfg)
    fb, ob = B.process_clip(np.ascontiguousarray(frames[5][None, k]), cfg)
    assert np.array_equal(fa[:, k], fb[:, 0]) and np.array_equal(oa[:, k], ob), "clip"
    for name, lv in state_names(B, O.MODE_LAPLACE):
        assert np.array_equal(A.get_state(name, lv)[k], B.get_state(name, lv)[0]), (name, lv)


def test_device_to_device():
    """Device 0 -> device 1, when two GPUs are visible."""
    if capi.lib().mc_device_count() < 2:
        pytest.skip("needs two GPUs")
    check_move(Move(O.MODE_PHASE, PHASE_UI, 96, 64, b_device=1, entries=ENTRIES[:4]))
    check_move(Move(O.MODE_COLOR, COLOR_UI, 96, 64, before=21, options=(("color_lane_lifecycle", 1),), b_device=1,
                    entries=ENTRIES[:4]))
