"""Plain-Python restatement of cv2.findContours(mask, RETR_CCOMP, CHAIN_APPROX_NONE | CHAIN_APPROX_SIMPLE), the call
mmdet.structures.mask.bitmap_to_polygon makes (mmdet/structures/mask/structures.py:1166-1194), written as the device
kernels in rsprompter_b200/csrc/contours.cu compute it: from connected components and one independent walk per border
instead of cv2's sequential raster scan.

The image is seen with a one-pixel zero border (cv2 treats everything outside the image as background).
- Outer borders: one per 8-connected foreground component, starting at its first pixel in raster order.
- Hole borders: one per 4-connected background component that does not reach the border, starting at the left
  neighbour of the hole's first pixel in raster order (always foreground).  Its parent is the outer border of the
  component that holds that start pixel.
- List order: outer borders by descending raster order of their start points, each followed by its holes, also by
  descending raster order of their start points.
- Each border is traced by cv2's border following (icvFetchContour): the initial neighbour search goes clockwise from
  the background pixel (left for an outer border, right for a hole), each later one counter-clockwise from the
  direction after the one it came in by.  CHAIN_APPROX_SIMPLE emits a point only where the direction of the move out of
  it differs from the previous move, which can drop the start point.
- Hierarchy (RETR_CCOMP's two levels): [next, prev, first_child, parent] with next / prev linking the outer borders
  among themselves and the holes of one outer border among themselves, in list order.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

CHAIN_APPROX_NONE = 1       # cv2's values
CHAIN_APPROX_SIMPLE = 2

# direction s = 0 .. 7: right, up-right, up, up-left, left, down-left, down, down-right as (dx, dy)
_DIRS = ((1, 0), (1, -1), (0, -1), (-1, -1), (-1, 0), (-1, 1), (0, 1), (1, 1))


def _walk(img: np.ndarray, y: int, x: int, hole: bool, approx: int) -> list:
    """cv2's border following from (y, x) of the zero-bordered image -> [(x, y)] in padded coordinates."""
    s = s_end = 0 if hole else 4
    while True:
        s = (s - 1) & 7
        y1, x1 = y + _DIRS[s][1], x + _DIRS[s][0]
        if img[y1, x1] or s == s_end:
            break
    if s == s_end and not img[y1, x1]:     # an isolated pixel
        return [(x, y)]
    pts = []
    cy, cx = y, x
    prev_s = s ^ 4
    while True:
        s_end = s
        while True:                        # counter-clockwise from the direction after the incoming one
            s += 1
            ny, nx = cy + _DIRS[s & 7][1], cx + _DIRS[s & 7][0]
            if img[ny, nx]:
                break
        s &= 7
        if s != prev_s or approx == CHAIN_APPROX_NONE:
            pts.append((cx, cy))
            prev_s = s
        if (ny, nx) == (y, x) and (cy, cx) == (y1, x1):
            break
        cy, cx = ny, nx
        s = (s + 4) & 7
    return pts


def find_contours(mask: np.ndarray, approx: int = CHAIN_APPROX_NONE) -> tuple:
    """mask [H, W] (nonzero = set) -> (contours: list of int32 [k, 2] (x, y), hierarchy int32 [1, n, 4] or None),
    cv2.findContours(mask.astype(np.uint8), cv2.RETR_CCOMP, approx)'s output."""
    H, W = mask.shape
    img = np.zeros((H + 2, W + 2), np.uint8)
    img[1:-1, 1:-1] = mask != 0
    fg, _ = ndimage.label(img, structure=np.ones((3, 3), int))
    bg, _ = ndimage.label(img == 0, structure=[[0, 1, 0], [1, 1, 1], [0, 1, 0]])
    Wp = W + 2
    flat_fg, flat_bg = fg.ravel(), bg.ravel()
    # first pixel of every component in raster order
    outer_start = {}
    for p in np.flatnonzero(flat_fg):
        outer_start.setdefault(int(flat_fg[p]), int(p))
    holes = {}                              # outer start -> [hole start]
    outside = int(flat_bg[0])               # the border's component
    seen = set()
    for p in np.flatnonzero(flat_bg):
        lab = int(flat_bg[p])
        if lab == outside or lab in seen:
            continue
        seen.add(lab)
        start = int(p) - 1
        holes.setdefault(outer_start[int(flat_fg[start])], []).append(start)
    contours, hier = [], []
    outers = sorted(outer_start.values(), reverse=True)
    prev_outer = -1
    for o in outers:
        oi = len(contours)
        if prev_outer >= 0:
            hier[prev_outer][0] = oi
        kids = sorted(holes.get(o, []), reverse=True)
        hier.append([-1, prev_outer, oi + 1 if kids else -1, -1])
        contours.append(_walk(img, o // Wp, o % Wp, False, approx))
        prev_outer = oi
        prev_kid = -1
        for h in kids:
            hi = len(contours)
            if prev_kid >= 0:
                hier[prev_kid][0] = hi
            hier.append([-1, prev_kid, -1, oi])
            contours.append(_walk(img, h // Wp, h % Wp, True, approx))
            prev_kid = hi
    out = [np.asarray(c, np.int32).reshape(-1, 2) - 1 for c in contours]
    return out, (np.asarray(hier, np.int32)[None] if hier else None)


def hierarchy_from_parents(parents: list) -> np.ndarray | None:
    """cv2's RETR_CCOMP hierarchy [1, n, 4] from the parent of every contour in list order (-1: an outer border)."""
    n = len(parents)
    if n == 0:
        return None
    hier = np.full((n, 4), -1, np.int32)
    last = {}                                # parent -> last contour seen with it
    for i, p in enumerate(parents):
        p = int(p)
        hier[i, 3] = p
        if p in last:
            hier[last[p], 0] = i
            hier[i, 1] = last[p]
        elif p >= 0:
            hier[p, 2] = i
        last[p] = i
    return hier[None]
