"""SURVEY.md §8f-3: ONE Motion (Laplace) stream cut into contiguous segments, one per rank, with the temporal state
handed from rank to rank through the linear recurrence (lvm_b200.shard.magnify_segment).  The sharded result must
equal the single-handle run of the whole clip up to f32 rounding of the carry (<= 1 LSB, >= 99.9 % identical).

CPU variants run the product's kernels on the CUDA-on-CPU emulation (tests/cuda_emu): in-process with a queue as the
transport, and as a real world_size-2 gloo job.  The `gpu` variant runs the same on an H100."""
import os
import socket

import numpy as np
import pytest

import lvm_b200 as L
from lvm_b200 import capi, shard
from lvm_b200.synth import synth_frame
from oracle import livim_oracle as O
from common import make_cfgs, u8_diff

W, H, LEVELS = 131, 75, 4


def clip(n):
    return [synth_frame(t, W, H, 3) for t in range(n)]


def single_stream(frames, cfg):
    proc = L.MagnificationProcessor(0)
    outs = [proc.process_image(f, cfg)[1] for f in frames]
    state = shard.export_motion_state(proc)
    proc.close()
    return outs, state


def check(outs, ref):
    assert len(outs) == len(ref)
    d = np.stack([u8_diff(a, b) for a, b in zip(outs, ref)])
    assert int(d.max()) <= 1 and float((d == 0).mean()) >= 0.999, (int(d.max()), float((d == 0).mean()))


def run_in_process(cuts, n, mode=O.MODE_LAPLACE, ui=(20, 50.0, 0.4, 3.0, 30, LEVELS), fps=30.0, size=(W, H), phase_tol=False):
    """all 'ranks' in this process, one after another, a dict as the transport"""
    cfg, _ = make_cfgs(mode, *ui, fps)
    frames = [synth_frame(t, size[0], size[1], 3, fps=fps) for t in range(n)]
    proc = L.MagnificationProcessor(0)
    ref = [proc.process_image(f, cfg) for f in frames]
    proc.close()
    bounds = [0] + list(cuts) + [n]
    world = len(bounds) - 1
    need = shard.preroll_frames(cfg)
    mailbox, outs = {}, []
    for rank in range(world):
        lo, hi = bounds[rank], bounds[rank + 1]
        outs += shard.magnify_segment(frames[lo:hi], cfg, rank, world, lambda: L.MagnificationProcessor(0),
                                      send=lambda flat, dst: mailbox.__setitem__(dst, flat.copy()),
                                      recv=lambda m, src, r=rank: mailbox.pop(r),
                                      preroll=frames[max(0, lo - need):lo] if rank else ())
    assert len(outs) == n
    for t, (o, (produced, r)) in enumerate(zip(outs, ref)):
        if not produced:                       # passthrough frames of the single stream (warm-up) come back as the input
            assert o is frames[t] or np.array_equal(o, frames[t]), t
            continue
        d = u8_diff(o, r)
        if phase_tol:
            assert int(d.max()) <= 3 and float((d == 0).mean()) >= 0.995, (t, int(d.max()), float((d == 0).mean()))
        else:
            assert int(d.max()) <= 1 and float((d == 0).mean()) >= 0.999, (t, int(d.max()), float((d == 0).mean()))


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


@pytest.mark.emu
@pytest.mark.parametrize("cuts,n", [((5,), 9), ((3, 4, 8), 10), ((1,), 3)])
def test_state_carry_in_process_on_emulation(emu, cuts, n):
    run_in_process(cuts, n)


@pytest.mark.emu
def test_color_segments_with_window_preroll_on_emulation(emu):
    """Color has a finite memory (the rolling window): pre-rolling window-1 frames reproduces the single stream; a cut
    inside the clip's own warm-up (fewer frames available than the window) and one in steady state."""
    run_in_process((6, 26), 34, mode=O.MODE_COLOR, ui=(100, 0.0, 0.8, 1.2, 0, 2), fps=8.0, size=(64, 48))


@pytest.mark.emu
def test_phase_segments_with_register_carry_on_emulation(emu):
    """Phase: two pre-roll frames (the reference's first frame leaves the prior pyramid without its Riesz pair) + the 3x3
    linear carry of (phase, r0, r1) per Butterworth filter and component; cuts at frame 1 (one pre-roll frame exists), 4, 7."""
    run_in_process((1, 4, 7), 11, mode=O.MODE_PHASE, ui=(50, 50.0, 0.4, 3.0, 0, 3), size=(96, 64), phase_tol=True)


@pytest.mark.emu
def test_carry_formula_reproduces_the_continuous_state(emu):
    """F = S + (1-c)^n (F_prev - B0) against the state of the uninterrupted run, plane by plane."""
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.0, 3.0, 30, LEVELS)     # coLow = 0 -> 0.01 (TemporalFilter.cpp:11)
    frames = clip(8)
    _, full = single_stream(frames, cfg)
    _, prev = single_stream(frames[:3], cfg)
    proc = L.MagnificationProcessor(0)
    proc.process_image(frames[3], cfg)
    b0 = shard.export_motion_state(proc)
    proc.set_option("analysis_only", 1)
    for f in frames[4:]:
        produced, out = proc.process_image(f, cfg)
        assert not produced and out is f                       # no frame is produced in the state-only pass
    end = shard.export_motion_state(proc)
    carried = shard.carry_motion_state(end, b0, prev, 5, cfg.magnification.coLow, cfg.magnification.coHigh)
    assert sorted(carried) == sorted(full) and len(full) == 2 * (LEVELS - 1)
    for k in full:
        err = float(np.abs(carried[k] - full[k]).max())
        assert err < 2e-5 * (float(np.abs(full[k]).max()) + 1.0), (k, err)
    proc.close()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, n, q):
    import sys
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import conftest
    conftest.use_emulated_library()
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, LEVELS)
    frames = clip(n)
    ids = shard.shard_streams(n, rank, world)                  # contiguous, balanced frame ranges
    send, recv = shard.dist_send_recv(dist, "cpu")
    outs = shard.magnify_segment([frames[i] for i in ids], cfg, rank, world, lambda: L.MagnificationProcessor(0), send, recv)
    q.put((rank, ids, np.stack(outs)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.emu
def test_state_carry_two_ranks_gloo(built):
    import torch.multiprocessing as mp
    world, n, port = 2, 9, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=300) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    try:
        cfg, _ = make_cfgs(O.MODE_LAPLACE, 20, 50.0, 0.4, 3.0, 30, LEVELS)
        ref, _ = single_stream(clip(n), cfg)
    finally:
        capi.LIB_PATH, capi._lib = saved
    assert [i for r in res for i in r[1]] == list(range(n))
    check([o for r in res for o in r[2]], ref)


@pytest.mark.gpu
@pytest.mark.parametrize("cuts,n", [((6,), 12), ((2, 5, 9), 12)])
def test_state_carry_on_gpu(cuts, n):
    run_in_process(cuts, n)


@pytest.mark.gpu
def test_color_and_phase_segments_on_gpu():
    run_in_process((6, 26), 34, mode=O.MODE_COLOR, ui=(100, 0.0, 0.8, 1.2, 0, 2), fps=8.0, size=(160, 120))
    run_in_process((1, 4, 7), 11, mode=O.MODE_PHASE, ui=(50, 50.0, 0.4, 3.0, 0, 3), size=(160, 120), phase_tol=True)


def test_preroll_requirements():
    for mode, ui, fps, want in ((O.MODE_LAPLACE, (20, 50.0, 0.4, 3.0, 0, 4), 30.0, 0), (O.MODE_PHASE, (50, 50.0, 0.4, 3.0, 0, 4), 30.0, 2),
                                (O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 3), 30.0, 63), (O.MODE_COLOR, (100, 0.0, 0.8, 1.2, 0, 3), 8.0, 15)):
        cfg, _ = make_cfgs(mode, *ui, fps)
        assert shard.preroll_frames(cfg) == want
