"""The export canvas's "Original" / "Processed" labels as an overlay of per-pixel tone maps (mc_set_overlay).

The reference exporter burns its labels into a split canvas (ExportRequest::textOverlay, Exporter.cpp:36-50, 53-88):
each label darkens a box with addWeighted(box, 0.35, black, 0.65, 0) and then draws white anti-aliased Hershey text
over it.  Both steps are pointwise and treat the three channels alike, so the labelled canvas is
``out[y, x, c] = T_yx(in[y, x, c])`` with one u8 -> u8 map T per pixel, the identity outside the labels.
export_labels() reads every T off the labels drawn with cv2 onto flat grey canvases, three grey levels at a time (one
per channel), and keeps the tight box of the changed pixels with the distinct maps as a palette.  The compose kernel then
applies them to every canvas it writes; the core itself draws no text and needs no OpenCV.

This module is the executable specification of that recipe (INTEGRATION.md §2b) and the only module of the package that
imports cv2, lazily, inside export_labels().
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

from . import capi

SPLIT_NONE, SPLIT_LEFT_RIGHT, SPLIT_TOP_BOTTOM = capi.MC_SPLIT_NONE, capi.MC_SPLIT_LEFT_RIGHT, capi.MC_SPLIT_TOP_BOTTOM
_MARGIN = 16   # pixels around a label's box that its anti-aliased strokes never reach (checked when the maps are read)


class Overlay:
    """Rects of u16 map indices on a canvas_w x canvas_h canvas and a palette of 256-byte maps.  Keeps its arrays alive
    for the ctypes struct (`struct`, for mc_set_overlay) and applies itself to BGR canvases in numpy (`apply`)."""

    def __init__(self, canvas_w: int, canvas_h: int, rects: Sequence[Tuple[int, int, np.ndarray]], palette: np.ndarray):
        self.canvas_w, self.canvas_h = int(canvas_w), int(canvas_h)
        self.rects = [(int(x), int(y), np.ascontiguousarray(idx, np.uint16)) for x, y, idx in rects]
        self.palette = np.ascontiguousarray(palette, np.uint8).reshape(-1, 256)
        if len(self.rects) > capi.MC_OVERLAY_MAX_RECTS:
            raise ValueError(f"at most {capi.MC_OVERLAY_MAX_RECTS} rects")
        st = capi.McOverlay()
        st.canvas_w, st.canvas_h, st.rects = self.canvas_w, self.canvas_h, len(self.rects)
        for i, (x, y, idx) in enumerate(self.rects):
            st.rect[i] = capi.McOverlayRect(x, y, idx.shape[1], idx.shape[0], idx.ctypes.data)
        st.maps, st.map = len(self.palette), self.palette.ctypes.data
        self.struct = st

    def boxes(self) -> List[Tuple[int, int, int, int]]:
        """(x, y, w, h) of every rect"""
        return [(x, y, idx.shape[1], idx.shape[0]) for x, y, idx in self.rects]

    def apply(self, canvas: np.ndarray) -> np.ndarray:
        """The labelled copy of a canvas_h x canvas_w BGR canvas: map[index][v] per channel inside each rect."""
        if canvas.shape[:2] != (self.canvas_h, self.canvas_w):
            raise ValueError(f"canvas is {canvas.shape[1]} x {canvas.shape[0]}, the overlay {self.canvas_w} x {self.canvas_h}")
        out = canvas.copy()
        for x, y, idx in self.rects:
            h, w = idx.shape
            sub = out[y:y + h, x:x + w]
            out[y:y + h, x:x + w] = self.palette[idx[..., None].astype(np.intp), sub]
        return out


def _lround(v: float) -> int:
    """std::lround: halves away from zero (v >= 0 here)"""
    f = math.floor(v)
    return int(f) + (1 if v - f >= 0.5 else 0)


def _label_box(cv2, text: str, x: int, y: int, scale: float):
    """drawLabel's geometry (Exporter.cpp:36-50) -> (box x, y, w, h before clipping, thickness, text origin)"""
    thickness = max(1, _lround(scale))
    (tw, th), baseline = cv2.getTextSize(text, cv2.FONT_HERSHEY_SIMPLEX, scale, thickness)
    pad = max(2, _lround(scale * 4))
    return (x, y, tw + 2 * pad, th + baseline + 2 * pad), thickness, (x + pad, y + pad + th)


def export_labels(canvas_w: int, canvas_h: int, split: int) -> Overlay:
    """The exporter's labels on a canvas_w x canvas_h canvas of `split` (mc_compose_geometry's canvas) as an Overlay.
    No labels (zero rects) for SPLIT_NONE."""
    if canvas_w < 1 or canvas_h < 1 or split not in (SPLIT_NONE, SPLIT_LEFT_RIGHT, SPLIT_TOP_BOTTOM):
        raise ValueError("canvas size < 1 or split out of range")
    identity = np.arange(256, dtype=np.uint8)[None]
    if split == SPLIT_NONE:
        return Overlay(canvas_w, canvas_h, [], identity)
    import cv2

    w, h = (canvas_w // 2, canvas_h) if split == SPLIT_LEFT_RIGHT else (canvas_w, canvas_h // 2)
    scale = min(max(w / 800.0, 0.4), 1.5)
    labels = [("Original", 6, 6), ("Processed", w + 6, 6) if split == SPLIT_LEFT_RIGHT else ("Processed", 6, h + 6)]
    drawn = []   # (text, box clipped to the canvas, thickness, origin, band with margin)
    for text, x, y in labels:
        (bx, by, bw, bh), thickness, org = _label_box(cv2, text, x, y, scale)
        x0, y0, x1, y1 = max(bx, 0), max(by, 0), min(bx + bw, canvas_w), min(by + bh, canvas_h)
        if x1 <= x0 or y1 <= y0:
            continue   # drawLabel returns before it draws
        band = (max(x0 - _MARGIN, 0), max(y0 - _MARGIN, 0), min(x1 + _MARGIN, canvas_w), min(y1 + _MARGIN, canvas_h))
        drawn.append((text, (x0, y0, x1, y1), thickness, org, band))
    # labels whose bands meet are drawn together, in order, onto one band (their boxes may overlap)
    groups: List[list] = []
    for d in drawn:
        b = d[4]
        if groups and any(o[4][0] < b[2] and b[0] < o[4][2] and o[4][1] < b[3] and b[1] < o[4][3] for o in groups[-1]):
            groups[-1].append(d)
        else:
            groups.append([d])
    rects, maps = [], []
    for g in groups:
        bx0, by0 = min(d[4][0] for d in g), min(d[4][1] for d in g)
        bx1, by1 = max(d[4][2] for d in g), max(d[4][3] for d in g)
        t = _band_maps(cv2, g, scale, bx0, by0, bx1 - bx0, by1 - by0)   # [256, band h, band w]
        changed = (t != identity.reshape(256, 1, 1)).any(0)
        # strokes reaching a band edge inside the canvas would be cut there but not on the canvas
        inner = [changed[:, 0] if bx0 > 0 else None, changed[:, -1] if bx1 < canvas_w else None,
                 changed[0] if by0 > 0 else None, changed[-1] if by1 < canvas_h else None]
        assert not any(e is not None and e.any() for e in inner), "a label reaches the edge of its band"
        ys, xs = np.nonzero(changed)
        if len(ys) == 0:
            continue
        y0, y1, x0, x1 = ys.min(), ys.max() + 1, xs.min(), xs.max() + 1
        rects.append((bx0 + x0, by0 + y0, (y1 - y0, x1 - x0)))
        maps.append(t[:, y0:y1, x0:x1].reshape(256, -1).T)
    if not rects:
        return Overlay(canvas_w, canvas_h, [], identity)
    rows = np.ascontiguousarray(np.concatenate(maps))
    first = {}   # map bytes -> palette entry, in order of first use
    inverse = np.fromiter((first.setdefault(r, len(first)) for r in map(bytes, rows)), np.uint16, len(rows))
    palette = np.frombuffer(b"".join(first), np.uint8).reshape(-1, 256)
    out, k = [], 0
    for x, y, shape in rects:
        n = shape[0] * shape[1]
        out.append((x, y, inverse[k:k + n].reshape(shape)))
        k += n
    return Overlay(canvas_w, canvas_h, out, palette)


def _band_maps(cv2, group, scale, bx, by, bw, bh) -> np.ndarray:
    """drawLabel of each label in the group, in order, on a bw x bh band at (bx, by) of the canvas filled with each grey
    level (three per drawing, one per channel) -> T[v] as [256][bh][bw] u8"""
    t = np.empty((258, bh, bw), np.uint8)
    for v in range(0, 258, 3):
        band = np.empty((bh, bw, 3), np.uint8)
        band[:] = np.minimum(np.arange(v, v + 3), 255).astype(np.uint8)
        for text, (x0, y0, x1, y1), thickness, (ox, oy), _ in group:
            roi = band[y0 - by:y1 - by, x0 - bx:x1 - bx]
            roi[:] = cv2.addWeighted(roi, 0.35, np.zeros_like(roi), 0.65, 0.0)
            cv2.putText(band, text, (ox - bx, oy - by), cv2.FONT_HERSHEY_SIMPLEX, scale, (255, 255, 255), thickness,
                        cv2.LINE_AA)
        t[v:v + 3] = band.transpose(2, 0, 1)
    return t[:256]
