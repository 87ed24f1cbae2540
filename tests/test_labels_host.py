"""The export labels as an overlay of tone maps (lvm_b200.labels), pinned to the reference's own compose().

export_labels(canvas_w, canvas_h, split) applied to compose_oracle.compose(o, p, split) must equal, bit for bit, the
canvas the reference exporter burns its labels into: Exporter.cpp's compose(o, p, split, overlay = true), compiled in
place into oracle/_ref/_exporter_ref (oracle/exporter_ref).  Covered: every even pane width from 2 to 1300 (the 0.4
clamp below 320, thickness 1 below 1200, thickness 2 from 1200), 1920 and 3840, heights that clip the label boxes and
heights that do not, boxes clipped by the canvas, and narrow panes where "Original" runs into the second pane and over
"Processed".  CPU only; skipped, as test_ref_pin.py is, when _exporter_ref is neither built nor buildable."""
import os
import time

import numpy as np
import pytest

from lvm_b200 import capi
from lvm_b200.labels import export_labels
from compose_oracle import compose
from oracle.exporter_ref import build as exporter_ref

R = exporter_ref.load()
if R is None and os.environ.get("MC_REQUIRE_REF") == "1":
    raise RuntimeError("MC_REQUIRE_REF=1 but oracle/_ref/_exporter_ref is missing")
needs_ref = pytest.mark.skipif(R is None, reason="oracle/_ref/_exporter_ref is not built and /root/reference is absent")

LR, TB = capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM


def panes(w, h, seed):
    """random original / processed panes, one of them with a 0 and a 255 column band"""
    rng = np.random.default_rng(seed)
    o = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    p = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    p[:, : w // 3] = 0
    p[:, w // 3: 2 * w // 3] = 255
    return o, p


def check(w, h, split, seed=0, flat=True):
    o, p = panes(w, h, seed)
    cases = [(o, p)] + ([(np.zeros_like(o), np.full_like(p, 255)), (np.full_like(o, 255), np.zeros_like(p))] if flat else [])
    canvas = compose(o, p, split)
    ov = export_labels(canvas.shape[1], canvas.shape[0], split)
    for a, b in cases:
        want = R.compose(a, b, split, True)
        assert want is not None and np.array_equal(ov.apply(compose(a, b, split)), want), (w, h, split)
    return ov


def rects_are_tight_and_disjoint(ov):
    boxes = ov.boxes()
    assert len(boxes) <= capi.MC_OVERLAY_MAX_RECTS and 1 <= len(ov.palette) <= 65536
    for i, (x, y, w, h) in enumerate(boxes):
        assert 0 <= x and 0 <= y and x + w <= ov.canvas_w and y + h <= ov.canvas_h
        for (x2, y2, w2, h2) in boxes[:i]:
            assert not (x < x2 + w2 and x2 < x + w and y < y2 + h2 and y2 < y + h)
        idx = ov.rects[i][2]
        changed = (ov.palette[idx] != np.arange(256, dtype=np.uint8)).any(-1)   # [h][w]: not the identity
        assert changed[0].any() and changed[-1].any() and changed[:, 0].any() and changed[:, -1].any()


@needs_ref
@pytest.mark.parametrize("split", [LR, TB], ids=["left_right", "top_bottom"])
@pytest.mark.parametrize("h", [12, 40])
def test_every_even_width_to_1300(split, h):
    """h = 12 clips every box at the bottom (of the canvas for left/right, of the first pane's label into the second for
    top/bottom); h = 40 clips none below the 0.4 clamp"""
    for w in range(2, 1301, 2):
        rects_are_tight_and_disjoint(check(w, h, split, seed=w, flat=w % 64 == 0))


@needs_ref
@pytest.mark.parametrize("split", [LR, TB], ids=["left_right", "top_bottom"])
@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160), (1300, 17), (1200, 64), (1198, 64), (320, 20), (318, 8)])
def test_wide_panes_and_clipped_boxes(split, w, h):
    rects_are_tight_and_disjoint(check(w, h, split))


@needs_ref
@pytest.mark.parametrize("split", [LR, TB], ids=["left_right", "top_bottom"])
def test_narrow_panes_merge_overlapping_labels(split):
    """Narrow panes: "Original" runs into the second pane; where the two boxes meet they are one rect"""
    merged = 0
    for w in range(2, 120, 2):
        ov = check(w, 30 if split == LR else 8, split, seed=w)
        rects_are_tight_and_disjoint(ov)
        merged += len(ov.boxes()) == 1
    assert merged > 0


def test_split_none_has_no_rects():
    ov = export_labels(640, 360, capi.MC_SPLIT_NONE)
    assert ov.boxes() == [] and ov.struct.rects == 0 and len(ov.palette) == 1
    img = np.random.default_rng(1).integers(0, 256, (360, 640, 3), dtype=np.uint8)
    assert np.array_equal(ov.apply(img), img)


def test_struct_matches_arrays():
    ov = export_labels(3840, 1080, LR)
    st = ov.struct
    assert (st.canvas_w, st.canvas_h, st.rects, st.maps) == (3840, 1080, len(ov.rects), len(ov.palette))
    for i, (x, y, idx) in enumerate(ov.rects):
        r = st.rect[i]
        assert (r.x, r.y, r.w, r.h, r.index) == (x, y, idx.shape[1], idx.shape[0], idx.ctypes.data)
    assert st.map == ov.palette.ctypes.data and ov.palette.shape[1] == 256


@pytest.mark.parametrize("split", [LR, TB], ids=["left_right", "top_bottom"])
def test_builder_time_at_two_4k_panes(split):
    """The builder runs once per export geometry on the CPU: well under a second for two 4K panes"""
    cw, ch = (7680, 2160) if split == LR else (3840, 4320)
    t = time.perf_counter()
    ov = export_labels(cw, ch, split)
    dt = time.perf_counter() - t
    print(f"export_labels({cw}, {ch}): {dt * 1e3:.0f} ms, {sum(w * h for *_, w, h in ov.boxes())} px, {len(ov.palette)} maps")
    assert len(ov.boxes()) == 2 and dt < 1.0
