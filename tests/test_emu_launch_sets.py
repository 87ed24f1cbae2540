"""Which kernels each call launches, on the CUDA-on-CPU emulation (tests/cuda_emu): a fixed script of frame and clip calls
with profile_kernels on, and after every call the exact composition {(kernel, level): launches} it recorded.  Frame and
clip calls share their host orchestration, so this pins the launch sequence of every path the script reaches."""
import pytest

from lvm_b200 import capi
from oracle import livim_oracle as O
from common import make_cfgs
from test_gpu_clip import clip_frames, laplace_ui, run_clip, run_frames
from test_gpu_lanes import PHASE_UI, proc

pytestmark = pytest.mark.emu

W, H = 83, 45


@pytest.fixture()
def emu():
    import conftest
    saved = (capi.LIB_PATH, capi._lib)
    conftest.use_emulated_library()
    yield
    capi.LIB_PATH, capi._lib = saved


def run_script(mode, ui, c, steps, lanes=1, options=()):
    """`steps`: ("frame", None) one frame call, ("clip", n) one clip, ("restart", k) / ("hold", k) a lane's lifecycle.
    -> the composition recorded by each frame or clip call, in order."""
    cfg, _ = make_cfgs(mode, *ui)
    p = proc(lanes, (("profile_kernels", 1),) + tuple(options))
    got, t = [], 0
    for kind, arg in steps:
        if kind == "restart":
            p.restart_lane(arg)
            continue
        if kind == "hold":
            p.hold_lane(arg)
            continue
        n = 1 if kind == "frame" else arg
        fr = clip_frames(t, n, lanes, W, H, c)
        run_frames(p, fr, cfg) if kind == "frame" else run_clip(p, fr, cfg)
        got.append({k: v[0] for k, v in p.profile_read().items()})
        t += n
    p.close()
    return got


FRAMES_THEN_CLIP = [("frame", None), ("frame", None), ("clip", 3)]
ANALYSIS_ONLY = [("frame", None), ("clip", 3), ("frame", None)]
# a 3-lane handle: lane 2 restarted and lane 1 held for a frame call, then lane 2 restarted again for a clip
LANES = [("frame", None), ("restart", 2), ("hold", 1), ("frame", None), ("restart", 2), ("clip", 3)]

LAPLACE_CASES = {
    "color": (3, FRAMES_THEN_CLIP, 1, (), [
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("egress", 0): 1},
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("collapse", 2): 1, ("egress", 0): 1},
        {("ingest_lab", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1, ("collapse", 2): 1,
         ("egress", 0): 1},
    ]),
    "gray": (1, FRAMES_THEN_CLIP, 1, (), [
        {("down", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("egress", 0): 1},
        {("down", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("collapse", 2): 1, ("egress", 0): 1},
        {("down", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1, ("collapse", 2): 1,
         ("egress", 0): 1},
    ]),
    "color_analysis_only": (3, ANALYSIS_ONLY, 1, (("analysis_only", 1),), [
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("egress", 0): 1},
        {("ingest_lab", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1},
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1},
    ]),
    "gray_analysis_only": (1, ANALYSIS_ONLY, 1, (("analysis_only", 1),), [
        {("down", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("egress", 0): 1},
        {("down", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1},
        {("down", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1},
    ]),
    "color_analysis_only_first_clip": (3, [("clip", 3)], 1, (("analysis_only", 1),), [
        {("ingest_lab", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1, ("egress", 0): 1},
    ]),
    "color_lanes": (3, LANES, 3, (), [
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("egress", 0): 1},
        {("ingest_lab", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("collapse", 2): 1, ("egress", 0): 1},
        {("ingest_lab", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1, ("collapse", 2): 1,
         ("egress", 0): 1},
    ]),
    "color_lanes_faithful_level0": (3, LANES, 3, (("faithful_level0", 1),), [
        {("lab16", 0): 1, ("level", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("copy", 4): 2,
         ("egress", 0): 1},
        {("lab16", 0): 1, ("level", 0): 1, ("level", 1): 1, ("level", 2): 1, ("level", 3): 1, ("copy", 4): 2,
         ("collapse", 2): 1, ("egress", 0): 1},
        {("lab16", 0): 1, ("level_clip", 0): 1, ("level_clip", 1): 1, ("level_clip", 2): 1, ("level_clip", 3): 1,
         ("copy", 4): 2, ("collapse", 2): 1, ("egress", 0): 1},
    ]),
}


@pytest.mark.parametrize("case", list(LAPLACE_CASES))
def test_laplace_launch_sets(emu, case):
    c, steps, lanes, options, want = LAPLACE_CASES[case]
    assert run_script(O.MODE_LAPLACE, laplace_ui(4), c, steps, lanes, options) == want


PHASE_FRAME = {("lab16", 0): 1, ("riesz_analysis", 0): 1, ("riesz_analysis", 1): 1, ("riesz_phase", 0): 1,
               ("riesz_phase", 1): 1, ("riesz_amplify", 0): 1, ("riesz_amplify", 1): 1, ("riesz_collapse", 0): 1,
               ("riesz_collapse", 1): 1, ("riesz_egress", 0): 1}
PHASE_CLIP = {("lab16", 0): 1, ("riesz_analysis", 0): 1, ("riesz_analysis", 1): 1, ("riesz_phase_clip", 0): 1,
              ("riesz_phase_clip", 1): 1, ("riesz_amplify", 0): 1, ("riesz_amplify", 1): 1, ("riesz_collapse", 0): 1,
              ("riesz_collapse", 1): 1, ("riesz_egress", 0): 1}


def test_phase_launch_sets(emu):
    """3 levels: the first frame passes through after the analysis; a clip on a fresh handle holds that first frame"""
    first = {("lab16", 0): 1, ("riesz_analysis", 0): 1, ("riesz_analysis", 1): 1}
    assert run_script(O.MODE_PHASE, PHASE_UI, 3, FRAMES_THEN_CLIP) == [first, PHASE_FRAME, PHASE_CLIP]
    assert run_script(O.MODE_PHASE, PHASE_UI, 3, [("clip", 3), ("clip", 3)]) == [PHASE_CLIP, PHASE_CLIP]
