"""Greedy non-maximum merging without a GPU: the restatement (oracle.restate_nmm) on hand-worked examples and against
a plain double loop, the argument refusals of the greedy_nmm merge (they run before any launch), the CLI flags, and
that the new kernels do not spill."""
import os
import re
import sys

import numpy as np
import pytest
import torch

from oracle import restate_nmm as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tile(boxes, scores, labels):
    return dict(bboxes=torch.tensor(boxes, dtype=torch.float32), scores=torch.tensor(scores, dtype=torch.float32),
                labels=torch.tensor(labels))


def _one(boxes, scores, labels, thr, metric):
    return R.greedy_nmm(torch.tensor(boxes, dtype=torch.float32), torch.tensor(scores, dtype=torch.float32),
                        torch.tensor(labels), thr, metric)


def test_fragment_and_whole_object_merge_to_the_union_box():
    # a field from x 900 to 1300: tile 0 (window x < 1024) sees the fragment up to its edge, tile 1 at x 768 all of it
    t0 = _tile([[900, 100, 1024, 200]], [0.9], [4])
    t1 = _tile([[132, 100, 532, 200]], [0.7], [4])
    merged, groups = R.merge_results_by_nmm([t0, t1], [(0, 0), (768, 0)], (1024, 2048), 0.5, "ios", patch=1024)
    assert groups == [[0, 1]]
    assert merged["bboxes"].tolist() == [[900.0, 100.0, 1300.0, 200.0]]
    assert merged["scores"].tolist() == [pytest.approx(0.9)] and merged["labels"].tolist() == [4]
    # the hard merge keeps only the fragment
    from oracle.restate_large_image import merge_results_by_nms
    hard, keep = merge_results_by_nms([t0, t1], [(0, 0), (768, 0)], (1024, 2048), 0.25, patch=1024)
    assert keep.tolist() == [0] and hard["bboxes"].tolist() == [[900.0, 100.0, 1024.0, 200.0]]


def test_adjacent_distinct_objects_are_not_merged():
    for metric in ("ios", "iou"):
        assert _one([[0, 0, 100, 100], [100, 0, 200, 100]], [0.9, 0.8], [1, 1], 0.5, metric) == [[0], [1]]


def test_ios_and_iou_disagree():
    boxes = [[0, 0, 100, 100], [10, 10, 30, 30]]            # ios 1, iou 400 / 10000
    assert _one(boxes, [0.9, 0.8], [1, 1], 0.5, "ios") == [[0, 1]]
    assert _one(boxes, [0.9, 0.8], [1, 1], 0.5, "iou") == [[0], [1]]


def test_different_labels_never_merge():
    for metric in ("ios", "iou"):
        assert _one([[0, 0, 10, 10], [0, 0, 10, 10]], [0.9, 0.8], [1, 2], 0.0, metric) == [[0], [1]]


def test_value_exactly_at_the_threshold_matches():
    # ios: inter 2 over the smaller area 4
    assert _one([[0, 0, 4, 1], [2, 0, 6, 1]], [0.9, 0.8], [0, 0], 0.5, "ios") == [[0, 1]]
    assert _one([[0, 0, 4, 1], [2, 0, 6, 1]], [0.9, 0.8], [0, 0], np.nextafter(np.float32(0.5), 1), "ios") == [[0], [1]]
    # iou: inter 1 over the union 4
    assert _one([[0, 0, 3, 1], [2, 0, 4, 1]], [0.9, 0.8], [0, 0], 0.25, "iou") == [[0, 1]]
    assert _one([[0, 0, 3, 1], [2, 0, 4, 1]], [0.9, 0.8], [0, 0], 0.2500001, "iou") == [[0], [1]]


def test_zero_area_box():
    boxes = [[0, 0, 10, 10], [5, 5, 5, 10]]                 # the second has width 0: inter 0
    assert _one(boxes, [0.9, 0.8], [0, 0], 0.0, "ios") == [[0], [1]]       # 0 / 0 is NaN: no match even at 0
    assert _one(boxes, [0.9, 0.8], [0, 0], 0.0, "iou") == [[0, 1]]         # 0 / 100 = 0 >= 0
    assert _one(boxes, [0.9, 0.8], [0, 0], 0.01, "iou") == [[0], [1]]


def test_chain_is_not_transitive():
    # A-B and B-C match (iou 20 / 180), A-C do not overlap: C stays its own keeper
    boxes = [[0, 0, 10, 10], [8, 0, 18, 10], [16, 0, 26, 10]]
    assert _one(boxes, [0.9, 0.8, 0.7], [0, 0, 0], 0.1, "iou") == [[0, 1], [2]]
    merged = R.merge_groups(torch.tensor(boxes, dtype=torch.float32), torch.tensor([0.9, 0.8, 0.7]),
                            torch.tensor([0, 0, 0]), [[0, 1], [2]])
    assert merged["bboxes"].tolist() == [[0, 0, 18, 10], [16, 0, 26, 10]]
    # with B first, B absorbs both
    assert _one(boxes, [0.8, 0.9, 0.7], [0, 0, 0], 0.1, "iou") == [[1, 0, 2]]


def test_score_ties_go_by_tile_then_slot():
    t0 = _tile([[10, 10, 50, 50], [10, 10, 50, 50]], [0.5, 0.5], [0, 0])
    t1 = _tile([[0, 0, 50, 50]], [0.5], [0])                    # the same object in the next tile, scene x 10..60
    merged, groups = R.merge_results_by_nmm([t1, t0], [(10, 10), (0, 0)], (512, 512), 0.5, "ios")
    assert groups == [[0, 1, 2]]                                   # tile order of the call, then slot
    assert merged["bboxes"].tolist() == [[10.0, 10.0, 60.0, 60.0]]
    # which of the tied chain A-B-C is first decides the groups
    a, b, c = [0, 0, 10, 10], [8, 0, 18, 10], [16, 0, 26, 10]
    _, groups = R.merge_results_by_nmm([_tile([a, b, c], [0.5] * 3, [0] * 3)], [(0, 0)], (64, 64), 0.1, "iou")
    assert groups == [[0, 1], [2]]
    _, groups = R.merge_results_by_nmm([_tile([b, a, c], [0.5] * 3, [0] * 3)], [(0, 0)], (64, 64), 0.1, "iou")
    assert groups == [[0, 1, 2]]
    _, groups = R.merge_results_by_nmm([_tile([a], [0.5], [0]), _tile([b, c], [0.5] * 2, [0] * 2)], [(0, 0), (0, 0)],
                                       (64, 64), 0.1, "iou")
    assert groups == [[0, 1], [2]]


def test_score_thr_drops_candidates_first():
    t = _tile([[0, 0, 10, 10], [0, 0, 12, 12]], [0.2, 0.9], [0, 0])
    merged, groups = R.merge_results_by_nmm([t], [(0, 0)], (64, 64), 0.5, "ios", score_thr=0.5)
    assert groups == [[1]] and merged["bboxes"].tolist() == [[0, 0, 12, 12]]


def _literal(boxes, scores, labels, thr, metric):
    """The grouping as two plain Python loops over fp32 scalars."""
    f = np.float32
    order = sorted(range(len(scores)), key=lambda i: (-scores[i], i))
    absorbed, groups = set(), []
    for p, i in enumerate(order):
        if i in absorbed:
            continue
        g = [i]
        for j in order[p + 1:]:
            if j in absorbed or labels[j] != labels[i]:
                continue
            a, b = boxes[i], boxes[j]
            with np.errstate(invalid="ignore", divide="ignore"):
                w = max(f(0), f(min(a[2], b[2]) - max(a[0], b[0])))
                h = max(f(0), f(min(a[3], b[3]) - max(a[1], b[1])))
                inter = f(w * h)
                sa, sb = f(f(a[2] - a[0]) * f(a[3] - a[1])), f(f(b[2] - b[0]) * f(b[3] - b[1]))
                v = f(inter / f(f(sa + sb) - inter)) if metric == "iou" else f(inter / min(sa, sb))
            if v >= f(thr):
                absorbed.add(j)
                g.append(j)
        groups.append(g)
    return groups


@pytest.mark.parametrize("metric", ["ios", "iou"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_equals_the_literal_loops(metric, seed):
    g = np.random.default_rng(seed)
    n = 300
    xy = np.floor(g.uniform(0, 200, (n, 2))).astype(np.float32)
    wh = np.floor(g.uniform(0, 40, (n, 2))).astype(np.float32)
    boxes = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    scores = (np.round(g.uniform(0, 1, n) * 16) / 16).astype(np.float32)     # ties
    labels = g.integers(0, 3, n)
    for thr in (0.3, 0.5):
        got = R.greedy_nmm(torch.from_numpy(boxes), torch.from_numpy(scores), torch.from_numpy(labels), thr, metric)
        assert got == _literal(boxes, scores, labels, thr, metric)


# ------------------------------------------------------------------------------ refusals and the CLI
def test_bad_merge_arguments_raise_before_any_launch():
    from rsprompter_b200 import _lib
    from rsprompter_b200.large_image import merge_tile_records, predict_large_image
    n0 = _lib.launch_count
    with pytest.raises(ValueError, match="match metric 'dice'"):
        merge_tile_records([], [], (64, 64), nms_type="greedy_nmm", match_metric="dice")
    with pytest.raises(ValueError, match="merge nms type 'nmm'"):
        merge_tile_records([], [], (64, 64), nms_type="nmm")
    with pytest.raises(ValueError, match="match metric 'IOS'"):
        predict_large_image(None, None, merge_nms_type="greedy_nmm", merge_match_metric="IOS")
    with pytest.raises(ValueError, match="merge nms type 'greedy'"):
        predict_large_image(None, None, merge_nms_type="greedy")
    with pytest.raises(ValueError, match="match metric"):
        _lib.nmm_batched(None, None, None, 0.5, metric="giou")
    assert _lib.launch_count == n0


def test_cli_parses_the_merge_flags():
    from rsprompter_b200.large_image import build_parser
    ap = build_parser()
    a = ap.parse_args(["cfg.py", "scene.png", "--merge-nms-type", "greedy_nmm", "--merge-match-metric", "iou",
                       "--merge-iou-thr", "0.5"])
    assert (a.merge_nms_type, a.merge_match_metric, a.merge_iou_thr) == ("greedy_nmm", "iou", 0.5)
    a = ap.parse_args(["cfg.py", "scene.png"])
    assert (a.merge_nms_type, a.merge_match_metric) == ("nms", "ios")
    with pytest.raises(SystemExit):
        ap.parse_args(["cfg.py", "scene.png", "--merge-match-metric", "dice"])


def test_union_rle_rejects_bad_descriptors():
    import ctypes
    from rsprompter_b200 import _lib
    desc = (ctypes.c_int64 * 8)(2000, 3000, 0, 1, 2000, 3000, 1, 2)               # canvas 1 has parts 1 and 2
    good = (0, 128, 1024, 1024, 1024, 0, 0)
    fake = ctypes.c_void_p(16)                                    # never dereferenced: the checks precede every launch

    def status(part2, num_parts=3, d=desc):
        parts = (ctypes.c_int64 * 21)(*good, *good, *part2)
        return _lib._lib.rsp_mask_rle_union_lengths(fake, 1, fake, ctypes.cast(d, ctypes.c_void_p), 2, fake,
                                                    ctypes.cast(parts, ctypes.c_void_p), num_parts, fake, None)
    assert status((0, 128, 1024, 1024, 1024, 2000, 0)) == 1                     # origin below the canvas
    assert b"mask 1, part 2" in _lib._lib.rsp_last_error()
    assert status((0, 128, 1024, 1025, 1000, 0, 0)) == 1                        # more rows than the source has
    assert status((0, 128, 1024, 1000, 1000, 1500, 0)) == 1                     # leaves the canvas
    assert status(good, num_parts=2) == 1                                       # parts past num_parts
    assert b"outside the 2 parts" in _lib._lib.rsp_last_error()
    empty = (ctypes.c_int64 * 8)(2000, 3000, 0, 1, 2000, 3000, 1, 0)
    assert status(good, d=empty) == 1                                           # K = 0


# ------------------------------------------------------------------------------ ptxas
def _spills(log, pattern):
    out = {}
    for name, st, ld in re.findall(r"Function properties for (\S+)\s+\d+ bytes stack frame, (\d+) bytes spill stores, "
                                   r"(\d+) bytes spill loads", log):
        if re.search(pattern, name):
            out[name] = (int(st), int(ld))
    return out


def test_nmm_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    build = os.path.join(ROOT, "rsprompter_b200", "csrc", "build")
    with open(os.path.join(build, "detect.ptxas.log")) as f:
        det = _spills(f.read(), r"nmm_mask_kernel|nms_scan_kernel")
    with open(os.path.join(build, "rle.ptxas.log")) as f:
        rle = _spills(f.read(), r"mask_rle_union_kernel")
    assert len(det) == 4, sorted(det)                             # IoU, IoS; scan with and without owners
    assert len(rle) == 4, sorted(rle)                             # packed x write
    assert all(v == (0, 0) for v in {**det, **rle}.values()), {**det, **rle}
