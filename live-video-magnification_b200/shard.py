"""Multi-GPU plumbing for the replica-parallel path (SURVEY.md §8e): one process per GPU, every rank
serves its own independent streams.  The data path has NO per-frame collective; the only exchange is
a one-time broadcast of the POD parameter block from rank 0, plus a MAX-reduction of the timings for
reporting.  Works with any torch.distributed backend (NCCL on H100s, gloo in the CPU tests)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

from .capi import McParams


def bind_to_gpu_numa_node(device_index: int):
    """Pins the calling process to the CPUs of the NUMA node its GPU hangs off, so that the pinned frame buffers it
    allocates next are local to that GPU's PCIe root (one process per GPU: without this, ranks on a two-socket box
    stage half of their frames across the socket interconnect).  Returns (previous affinity, info dict) — restore with
    os.sched_setaffinity(0, previous) — or (None, {...reason}) when the topology cannot be read.  Linux sysfs only;
    never raises."""
    import os
    try:
        import torch
        pr = torch.cuda.get_device_properties(device_index)
        bus = f"{getattr(pr, 'pci_domain_id', 0):04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None, {"numa_node": None, "reason": "single NUMA node / not reported"}
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            spec = f.read().strip()
        cpus = set()
        for part in spec.split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        prev = os.sched_getaffinity(0)
        cpus &= prev
        if not cpus:
            return None, {"numa_node": node, "reason": "no allowed CPU on that node"}
        os.sched_setaffinity(0, cpus)
        return prev, {"numa_node": node, "cpus": len(cpus), "pci": bus}
    except Exception as e:   # noqa: BLE001 — topology is best effort
        return None, {"numa_node": None, "reason": repr(e)[:80]}


def shard_streams(total_streams: int, rank: int, world: int) -> List[int]:
    """Contiguous, balanced partition of stream ids 0..total-1 across ranks (weak scaling uses
    total = lanes_per_gpu * world so every rank gets exactly lanes_per_gpu)."""
    base, rem = divmod(total_streams, world)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


def params_to_bytes(p: McParams) -> bytes:
    return bytes(p)


def params_from_bytes(b: bytes) -> McParams:
    p = McParams()
    assert len(b) == C.sizeof(p)
    C.memmove(C.byref(p), b, C.sizeof(p))
    return p


def broadcast_params(p: Optional[McParams], dist=None, device="cpu", src: int = 0) -> McParams:
    """Rank `src` supplies p; everyone returns the same block (one NCCL / gloo broadcast)."""
    import torch
    n = C.sizeof(McParams)
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        assert p is not None
        return p
    buf = torch.zeros(n, dtype=torch.uint8, device=device)
    if dist.get_rank() == src:
        buf = torch.frombuffer(bytearray(params_to_bytes(p)), dtype=torch.uint8).to(device)
    dist.broadcast(buf, src=src)
    return params_from_bytes(bytes(buf.cpu().numpy().tobytes()))


def max_over_ranks(x: float, dist=None, device="cpu") -> float:
    import torch
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(x: float, dist=None, device="cpu") -> float:
    import torch
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


# --------------------------------------------------------------------------------------------------------------
# Temporal sharding of ONE stream (SURVEY.md §8f-3): exact state hand-off through the linear recurrence
# --------------------------------------------------------------------------------------------------------------
# All three modes (magnify_segment).  Motion (Laplace) keeps, per pyramid level and pixel, two exponential low-passes
#     hi_t = (1 - cH) hi_{t-1} + cH x_t ,   lo_t = (1 - cL) lo_{t-1} + cL x_t          (TemporalFilter.cpp:9-22)
# whose inputs x_t (the Laplacian bands of frame t) do not depend on the state, and a fresh stream starts with
# hi_0 = lo_0 = x_0 (MagnifyCore.hpp:98-103).  So if rank g processes its contiguous segment x_0 .. x_{n-1} as a
# fresh stream and ends in state S, the state the *continuous* run would have there is
#     F_g = S + (1 - c)^n (F_{g-1} - B_0)        with B_0 = x_0 (the state right after the segment's first frame)
# for each of the two filters.  That is the whole exchange: one state-sized message from rank g-1 to rank g
# (2 f32 planes per live level: 33 MB at 1080p, 133 MB at 4K), no per-frame collective.  Rank g then re-runs its
# segment from the true state F_{g-1}.  The first pass only needs the state, so it runs with option "analysis_only"
# (no synthesis / egress).  Results equal the single-handle run up to f32 rounding of the carry arithmetic.
_STATE_NAMES = ("lowpassHi", "lowpassLo")


def export_motion_state(proc, max_levels: int = 16):
    """-> {(name, level): ndarray [lanes][C][rows][cols]} for every state plane the handle keeps."""
    out = {}
    for name in _STATE_NAMES:
        for lvl in range(max_levels + 1):
            a = proc.get_state(name, lvl)
            if a is not None:
                out[(name, lvl)] = a
    return out


def import_state(proc, state) -> None:
    """{(name, level): planes} -> mc_set_state, for either mode's state planes."""
    for (name, lvl), a in state.items():
        proc.set_state(name, lvl, a)


import_motion_state = import_state   # earlier name


def carry_motion_state(end_state, first_state, prev_true_state, n_frames: int, co_low: float, co_high: float):
    """F_g = S + (1-c)^n (F_{g-1} - B_0), evaluated in float64 and rounded once to f32."""
    import numpy as np
    if co_low == 0:
        co_low = 0.01   # TemporalFilter.cpp:11-12
    decay = {"lowpassHi": (1.0 - co_high) ** n_frames, "lowpassLo": (1.0 - co_low) ** n_frames}
    out = {}
    for key, s in end_state.items():
        d = decay[key[0]]
        out[key] = (s.astype(np.float64) + d * (prev_true_state[key].astype(np.float64) - first_state[key].astype(np.float64))
                    ).astype(np.float32)
    return out


def _pack(state):
    import numpy as np
    keys = sorted(state)
    return keys, np.concatenate([state[k].ravel() for k in keys]) if keys else np.zeros(0, np.float32)


def _unpack(flat, like):
    out, pos = {}, 0
    for k in sorted(like):
        n = like[k].size
        out[k] = flat[pos:pos + n].reshape(like[k].shape).copy()
        pos += n
    return out


# Phase (Riesz): per band level and per component (cos / sin) the accumulated phase and the two Direct-Form-II
# registers of each Butterworth filter evolve linearly in their own state (TemporalFilter.cpp:340-351):
#     phase' = phase + d ;  y = B0 phase' + r0 ;  r0' = B1 phase' + r1 - A1 y ;  r1' = B2 phase' - A2 y
# i.e. x' = M x + v d with x = (phase, r0, r1) and the 3x3 matrix M below (d, the phase difference of the frame, depends
# only on the current and the previous frame's pyramids).  A fresh stream's first frame only initialises — and leaves the
# *prior* pyramid with a zeroed Riesz pair (RieszPyramid::init, RieszPyramid.cpp:196-213) — so a rank pre-rolls TWO frames:
# the first initialises, the second rebuilds the complete prior pyramid (and perturbs the registers: x_pre).  After the
# n frames of the segment the continuous run's state is x_local + M^n (x_true_start - x_pre).
# Color has a finite memory — the rolling window — so pre-rolling window-1 frames is exact and needs no message.
_RIESZ_REGS = ("r0", "r1")


def preroll_frames(cfg) -> int:
    """How many frames preceding its segment a rank needs (pass fewer only at the very start of the clip)."""
    from .processor import MagnificationMode, getOptimalBufferSize
    mode = int(cfg.magnification.mode)
    if mode == int(MagnificationMode.Color):
        return getOptimalBufferSize(int(cfg.magnification.framerate)) - 1
    return 2 if mode == int(MagnificationMode.Phase) else 0


def _riesz_matrix(a, b):
    import numpy as np
    return np.array([[1.0, 0.0, 0.0],
                     [b[1] - a[1] * b[0], -a[1], 1.0],
                     [b[2] - a[2] * b[0], -a[2], 0.0]], np.float64)


def export_riesz_state(proc, max_levels: int = 16):
    out = {}
    names = ["phase.c", "phase.s"] + [f"{f}.{r}.{c}" for f in ("lo", "hi") for r in _RIESZ_REGS for c in ("c", "s")]
    for lvl in range(max_levels):
        for name in names:
            a = proc.get_state(name, lvl)
            if a is not None:
                out[(name, lvl)] = a
    return out


def carry_riesz_state(end_state, first_state, prev_true_state, n_frames: int, co_low: float, co_high: float, framerate: float):
    """x_true_end = x_local_end + M^n (x_true_start - x_pre) per filter and component (x_pre = first_state: the local
    state after the pre-roll); the phase accumulator is shared by the two filters (first row of M is (1, 0, 0))."""
    import numpy as np
    from .processor import butterworth
    out = {}
    mats = {}
    for f, fc in (("lo", co_low), ("hi", co_high)):
        wn = 0.0 if framerate == 0.0 else fc / (framerate / 2.0)   # TemporalFilter.cpp:324-327
        a, b = butterworth(2, wn)
        mats[f] = np.linalg.matrix_power(_riesz_matrix(a, b), n_frames)
    levels = sorted({lvl for (_, lvl) in end_state})
    for lvl in levels:
        for c in ("c", "s"):
            def delta(name):
                return prev_true_state[(name, lvl)].astype(np.float64) - first_state[(name, lvl)].astype(np.float64)
            ph0 = delta(f"phase.{c}")
            out[(f"phase.{c}", lvl)] = (end_state[(f"phase.{c}", lvl)].astype(np.float64) + ph0).astype(np.float32)
            for f in ("lo", "hi"):
                x0 = [ph0, delta(f"{f}.r0.{c}"), delta(f"{f}.r1.{c}")]
                m = mats[f]
                for row, reg in ((1, "r0"), (2, "r1")):
                    corr = m[row, 0] * x0[0] + m[row, 1] * x0[1] + m[row, 2] * x0[2]
                    out[(f"{f}.{reg}.{c}", lvl)] = (end_state[(f"{f}.{reg}.{c}", lvl)].astype(np.float64) + corr).astype(np.float32)
    return out


def magnify_segment(frames, cfg, rank: int, world: int, make_processor, send, recv, preroll=()):
    """Temporal sharding of ONE stream: `frames` is rank `rank`'s contiguous segment of the clip (list of HxWxC uint8
    images), `preroll` the preroll_frames(cfg) frames that precede it in the clip (fewer at the clip's start, none for
    rank 0).  Returns the segment's magnified frames, equal — to f32 rounding of the carry (Motion, Phase) or of the
    ring position (Color) — to what a single handle processing the whole clip produces.

      Motion (Laplace): state-only first pass, one state message from rank-1, second pass from the true state.
      Phase (Riesz):    two pre-roll frames; first pass, one state message, second pass from the true registers.
      Color:            pre-roll of window-1 frames; no message at all.

    make_processor() -> MagnificationProcessor-like object (process_image / get_state / set_state / set_option / reset);
    send(flat_f32_array, dst_rank) / recv(n_floats, src_rank) move one flat f32 array between ranks (dist_send_recv
    wraps torch.distributed point-to-point).  Parameters must stay constant over the clip."""
    from .processor import MagnificationMode
    mode = int(cfg.magnification.mode)
    if not frames:
        raise ValueError("every rank needs at least one frame")
    preroll = list(preroll)
    p = cfg.magnification
    proc = make_processor()

    def run(seq):
        return [proc.process_image(f, cfg)[1] for f in seq]

    if mode == int(MagnificationMode.Color):
        run(preroll)
        outs = run(frames)
    elif mode == int(MagnificationMode.Laplace):
        if rank == 0:
            outs = run(frames)
            true_end = export_motion_state(proc)
        else:
            # pass 1: the segment as a fresh stream, state only
            proc.process_image(frames[0], cfg)
            first_state = export_motion_state(proc)
            proc.set_option("analysis_only", 1)
            run(frames[1:])
            end_state = export_motion_state(proc)
            prev_true = _unpack(recv(_pack(end_state)[1].size, rank - 1), end_state)
            true_end = carry_motion_state(end_state, first_state, prev_true, len(frames), p.coLow, p.coHigh)
        if rank + 1 < world:
            send(_pack(true_end)[1], rank + 1)
        if rank > 0:
            # pass 2: the segment again, continuing from the true state.  The first frame is processed once to set the
            # handle up (first-frame path), the state is replaced, and the same frame is processed again as frame n.
            proc.reset()
            proc.set_option("analysis_only", 0)
            proc.process_image(frames[0], cfg)
            import_state(proc, prev_true)
            outs = run(frames)
    elif mode == int(MagnificationMode.Phase):
        if rank > 0 and len(preroll) < 1:
            raise ValueError("Phase needs the (up to two) frames preceding the segment as pre-roll")
        if rank > 0:
            proc.set_option("analysis_only", 1)  # first pass: pyramids + filter registers only, no amplify / collapse / egress
        run(preroll[-2:])                       # frame 1 initialises (passthrough), frame 2 completes the prior pyramid
        first_state = export_riesz_state(proc)  # x_pre (all zero when there is a single pre-roll frame)
        outs = run(frames)                      # rank 0: final; rank > 0: first pass
        end_state = export_riesz_state(proc)
        if rank > 0:
            prev_true = _unpack(recv(_pack(end_state)[1].size, rank - 1), end_state)
            true_end = carry_riesz_state(end_state, first_state, prev_true, len(frames), p.coLow, p.coHigh, p.framerate)
        else:
            true_end = end_state
        if rank + 1 < world:
            send(_pack(true_end)[1], rank + 1)
        if rank > 0:
            proc.reset()
            proc.set_option("analysis_only", 0)
            run(preroll[-2:])
            import_state(proc, prev_true)
            outs = run(frames)
    else:
        raise NotImplementedError("mode None has nothing to shard")
    if hasattr(proc, "close"):
        proc.close()
    return outs


def dist_send_recv(dist, device="cpu"):
    """(send, recv) for magnify_segment over torch.distributed point-to-point (NCCL over NVLink with device='cuda',
    gloo on CPU)."""
    import numpy as np
    import torch

    def send(flat, dst):
        dist.send(torch.from_numpy(np.ascontiguousarray(flat)).to(device), dst=dst)

    def recv(n, src):
        t = torch.empty(n, dtype=torch.float32, device=device)
        dist.recv(t, src=src)
        return t.cpu().numpy()

    return send, recv
