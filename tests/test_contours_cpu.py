"""oracle.restate_contours (the construction csrc/contours.cu computes: borders from connected components, one
independent walk each) against cv2.findContours(RETR_CCOMP) in both approximation modes, exhaustively on small masks
and on seeded structured ones; the GeoJSON writer on given contours; the contours ABI's descriptor checks, which run
before any launch (fake device pointers are never dereferenced)."""
import itertools

import numpy as np
import pytest

from oracle.restate_contours import CHAIN_APPROX_NONE, CHAIN_APPROX_SIMPLE, find_contours, hierarchy_from_parents

cv2 = pytest.importorskip("cv2")

MODES = (CHAIN_APPROX_NONE, CHAIN_APPROX_SIMPLE)


def _check(mask, approx):
    c, h = cv2.findContours(np.ascontiguousarray(mask).astype(np.uint8), cv2.RETR_CCOMP, approx)
    rc, rh = find_contours(mask, approx)
    assert len(rc) == len(c), mask.astype(int)
    for a, b in zip(rc, c):
        assert np.array_equal(a, b.reshape(-1, 2)), (mask.astype(int), a, b.reshape(-1, 2))
    if h is None:
        assert rh is None
    else:
        assert np.array_equal(rh, h), (mask.astype(int), rh, h)
        assert np.array_equal(hierarchy_from_parents(rh[0, :, 3].tolist()), h)


def _every(h, w):
    codes = np.arange(1 << (h * w))
    return ((codes[:, None] >> np.arange(h * w)) & 1).astype(bool).reshape(-1, h, w)


@pytest.mark.parametrize("approx", MODES)
@pytest.mark.parametrize("hw", [(4, 4), (3, 5), (5, 3)])
def test_every_small_mask(hw, approx):
    for m in _every(*hw):
        _check(m, approx)


def _structured(seed):
    """Seeded masks up to 64 x 64: noise, 1-pixel lines, diagonal-only links, holes touching at corners, an island in
    a hole in an island, masks touching all four edges, empty and full."""
    rng = np.random.default_rng(seed)
    H, W = (int(v) for v in rng.integers(8, 65, 2))
    ys, xs = np.indices((H, W))
    out = [rng.random((H, W)) < d for d in (0.2, 0.4, 0.5, 0.6, 0.8)]
    out += [ys % 3 == 0, xs % 4 == 1, (ys == H // 2) | (xs == W // 3)]                       # lines
    out += [(ys + xs) % 2 == 0, (xs - ys) % 5 == 0]                                          # diagonal links only
    ring = np.ones((H, W), bool)
    ring[2:-2:3, 2:-2:3] = False                                                             # one-pixel holes
    ring[3:-2:3, 3:-2:3] = False                                                             # touching at corners
    out.append(ring)
    nest = np.zeros((H, W), bool)
    nest[1:-1, 1:-1] = True
    nest[3:-3, 3:-3] = False
    nest[5:-5, 5:-5] = True
    nest[6:-6, 6:-6] = False
    out.append(nest)                                                                         # island in hole in island
    edge = np.ones((H, W), bool)
    edge[H // 3:2 * H // 3, W // 3:2 * W // 3] = rng.random((2 * H // 3 - H // 3, 2 * W // 3 - W // 3)) < 0.5
    out += [edge, np.zeros((H, W), bool), np.ones((H, W), bool)]
    return out


@pytest.mark.parametrize("approx", MODES)
@pytest.mark.parametrize("seed", range(12))
def test_structured_masks(seed, approx):
    for m in _structured(seed):
        _check(m, approx)


# ---- GeoJSON -------------------------------------------------------------------------------------------------------
def test_geojson_rings_holes_and_degenerate_borders():
    from rsprompter_b200.geojson import feature_collection, multipolygon
    sq = np.array([[1, 1], [1, 4], [4, 4], [4, 1]], np.int32)
    hole = np.array([[2, 1], [1, 2], [2, 3], [3, 2]], np.int32)
    dot = np.array([[7, 7]], np.int32)
    line = np.array([[9, 0], [9, 3]], np.int32)
    hier = np.array([[[2, -1, 1, -1], [-1, -1, -1, 0], [3, 0, -1, -1], [-1, 2, -1, -1]]], np.int32)
    geo = multipolygon([sq, hole, dot, line], hier)
    closed = lambda a: a.tolist() + [a[0].tolist()]                                          # noqa: E731
    assert geo == dict(type="MultiPolygon", coordinates=[[closed(sq), closed(hole)]])
    # an outer border left out takes its holes with it; no valid ring at all -> null geometry
    h2 = np.array([[[1, -1, -1, -1], [-1, 0, 2, -1], [-1, -1, -1, 1]]], np.int32)
    assert multipolygon([dot, line, hole], h2) is None
    assert multipolygon([], None) is None
    fc = feature_collection([dict(score=0.5, bbox=[1, 2, 3, 4]), dict(score=0.25)],
                            [([sq, hole, dot, line], hier), ([], None)])
    assert fc["type"] == "FeatureCollection" and len(fc["features"]) == 2
    assert fc["features"][0] == dict(type="Feature", properties=dict(score=0.5, bbox=[1, 2, 3, 4]), geometry=geo)
    assert fc["features"][1]["geometry"] is None
    with pytest.raises(ValueError):
        feature_collection([dict()], [])


def test_geojson_from_the_oracle_contours_is_valid():
    """Rings from CHAIN_APPROX_SIMPLE contours: closed, at least 4 positions, holes inside their outer ring's box."""
    from rsprompter_b200.geojson import multipolygon
    for m in _structured(3):
        geo = multipolygon(*find_contours(m, CHAIN_APPROX_SIMPLE))
        if geo is None:
            continue
        for poly in geo["coordinates"]:
            xs, ys = zip(*poly[0])
            for ring in poly:
                assert ring[0] == ring[-1] and len(ring) >= 4
                assert all(min(xs) <= x <= max(xs) and min(ys) <= y <= max(ys) for x, y in ring)


# ---- ABI checks ----------------------------------------------------------------------------------------------------
P = 1 << 24                    # a fake, 16-byte aligned device pointer


def _call(desc, parts, approx=CHAIN_APPROX_NONE, ws_bytes=1 << 40):
    import ctypes

    from rsprompter_b200 import _lib
    d = np.ascontiguousarray(desc, np.int64)
    p = np.ascontiguousarray(parts, np.int64)
    st = _lib._lib.rsp_mask_contours_lengths(P, P, d.ctypes.data, len(d), P, p.ctypes.data, len(p), approx, P,
                                             ws_bytes, P, P, None)
    msg = (_lib._lib.rsp_last_error() or b"").decode()
    nb = ctypes.c_longlong(0)
    ws_st = _lib._lib.rsp_mask_contours_ws_bytes(d.ctypes.data, len(d), p.ctypes.data, len(p), ctypes.byref(nb))
    return st, msg, ws_st, nb.value


PART = (0, 8, 10, 10, 60, 5, 3)    # 10 rows of 8 bytes, visible 10 x 60 at (5, 3)


@pytest.mark.parametrize("desc, parts, what", [
    ([(0, 100, 0, 1)], [PART], "canvas 0 x 100"),
    ([(50000, 50000, 0, 1)], [PART], "canvas 50000 x 50000"),
    ([(100, 100, 0, 0)], [PART], "parts [0, 0 + 0)"),
    ([(100, 100, 1, 1)], [PART], "parts [1, 1 + 1)"),
    ([(100, 100, 0, 2)], [PART], "parts [0, 0 + 2)"),
    ([(100, 100, 0, 1)], [(0, 8, 10, 10, 60, 100, 3)], "origin (100, 3) outside"),
    ([(100, 100, 0, 1)], [(0, 8, 10, 10, 60, 95, 3)], "leaves the 100 x 100 canvas"),
    ([(100, 100, 0, 1)], [(0, 8, 10, 10, 65, 5, 3)], "exceeds the source"),
    ([(100, 100, 0, 1)], [(0, 8, 9, 10, 60, 5, 3)], "exceeds the source"),
    ([(100, 100, 0, 1)], [(-1, 8, 10, 10, 60, 5, 3)], "exceeds the source"),
])
def test_abi_rejects_bad_descriptors(desc, parts, what):
    st, msg, ws_st, _ = _call(desc, parts)
    assert st == 1 and what in msg, msg
    assert ws_st == 1


def test_abi_rejects_bad_approx_and_small_workspace():
    st, msg, ws_st, need = _call([(100, 100, 0, 1)], [PART], approx=3)
    assert st == 1 and "approx 3" in msg
    assert ws_st == 0 and need == 256 + 768 + 16 * 12 * 62         # header, bits, four int32 arrays of 12 x 62
    st, msg, _, _ = _call([(100, 100, 0, 1)], [PART], ws_bytes=need - 1)
    assert st == 1 and f"workspace of {need - 1} bytes, {need} needed" in msg, msg


# ---- ptxas ---------------------------------------------------------------------------------------------------------
def test_contour_kernels_do_not_spill():
    """Every kernel of csrc/contours.cu keeps its state in registers: no stack frame, no spills (ptxas -v report the
    Makefile keeps under csrc/build/)."""
    import os
    import re
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(root, "rsprompter_b200", "csrc", "build", "contours.ptxas.log")) as f:
        text = f.read()
    kernels = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'", text)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(kernels) == 8 and len(frames) == len(kernels), (kernels, frames)
    assert all(f == ("0", "0", "0") for f in frames), list(zip(kernels, frames))
