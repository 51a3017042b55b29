"""Soft-NMS without a GPU: the restated mmcv loop on hand-worked problems, the vectorised restatement and its removal
rule against the literal loop, NMS config parsing of the anchor heads, and what ptxas made of the new kernels."""
import copy
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

from oracle import restate_soft_nms as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _both(boxes, scores, **kw):
    """The literal loop and the vectorised one must agree bit for bit; returns the literal's result."""
    d1, i1 = R.soft_nms_literal(np.array(boxes, np.float32), np.array(scores, np.float32), **kw)
    d2, i2 = R.soft_nms(np.array(boxes, np.float32), np.array(scores, np.float32), **kw)
    assert np.array_equal(i1, i2) and np.array_equal(d1.view(np.int32), d2.view(np.int32))
    return d1, i1


def test_removal_below_min_score_moves_the_last_candidate_in():
    # 1 coincides with 0 (ovr 1, linear weight 0): removed, and 3 (the last) takes its slot before 2
    boxes = [[0, 0, 10, 10], [0, 0, 10, 10], [20, 20, 30, 30], [40, 40, 50, 50]]
    d, i = _both(boxes, [0.9, 0.8, 0.5, 0.7], iou_threshold=0.3, min_score=0.001, method="linear")
    assert i.tolist() == [0, 3, 2]
    assert d[:, 4].tolist() == [f32(0.9), f32(0.7), f32(0.5)]


def test_removal_order_decides_a_tie():
    # 1 and 3 tie at 0.7; 1 is removed at step 0 and the last candidate (3) moves into its slot, ahead of 2 (0.7 too)
    boxes = [[0, 0, 10, 10], [0, 0, 10, 10], [20, 20, 30, 30], [40, 40, 50, 50]]
    d, i = _both(boxes, [0.9, 0.8, 0.7, 0.7], iou_threshold=0.3, min_score=0.001, method="linear")
    assert i.tolist() == [0, 3, 2]


def test_equal_scores_first_position_wins_and_a_swap_reorders():
    boxes = [[0, 0, 1, 1], [10, 10, 11, 11], [20, 20, 21, 21]]
    _, i = _both(boxes, [0.5, 0.5, 0.9])
    assert i.tolist() == [2, 1, 0]            # 2 swaps into position 0, so 1 now precedes 0
    _, i = _both(boxes, [0.5, 0.5, 0.4])
    assert i.tolist() == [0, 1, 2]            # plain tie: the first position wins


@pytest.mark.parametrize("method", ["naive", "linear", "gaussian"])
def test_overlap_exactly_at_the_threshold(method):
    # areas 3 and 2, intersection 1, union 4: ovr == 0.25 exactly
    boxes = [[0, 0, 3, 1], [2, 0, 4, 1]]
    d, i = _both(boxes, [0.9, 0.8], iou_threshold=0.25, sigma=0.5, min_score=0.001, method=method)
    if method == "naive":
        assert i.tolist() == [0]
    elif method == "linear":
        assert i.tolist() == [0, 1] and d[1, 4] == f32(0.8) * f32(0.75)
    else:
        w = f32(math.exp(float(f32(-(f32(0.25) * f32(0.25))) / f32(0.5))))
        assert i.tolist() == [0, 1] and d[1, 4] == f32(0.8) * w
    # just below the threshold linear and naive leave the score alone
    d, i = _both(boxes, [0.9, 0.8], iou_threshold=0.2500001, method=method)
    if method != "gaussian":
        assert i.tolist() == [0, 1] and d[1, 4] == f32(0.8)


def test_every_score_below_min_score():
    # the first selection is made whatever its score; the rest fall below min_score and are removed
    d, i = _both([[0, 0, 1, 1], [5, 5, 6, 6], [9, 9, 10, 10]], [0.0005, 0.0002, 0.0007], min_score=0.001)
    assert i.tolist() == [2] and d[0, 4] == f32(0.0007)


def test_single_candidate():
    d, i = _both([[1, 2, 3, 4]], [0.25])
    assert i.tolist() == [0] and d.tolist() == [[1, 2, 3, 4, 0.25]]


def test_classes_are_separated_by_the_offset():
    b = torch.tensor([[0, 0, 10, 10], [0, 0, 10, 10], [0, 0, 10, 10]], dtype=torch.float32)
    s = torch.tensor([0.9, 0.8, 0.7])
    dets, keep = R.batched_nms(b, s, torch.tensor([0, 1, 0]), dict(type="soft_nms", iou_threshold=0.5))
    assert keep.tolist() == [0, 1] and dets[:, 4].tolist() == [s[0].item(), s[1].item()]
    assert torch.equal(dets[:, :4], b[:2])


def _random_problem(rng, n, ties):
    xy = rng.uniform(0, 200, (n, 2)).astype(np.float32)
    wh = rng.uniform(0, 40, (n, 2)).astype(np.float32)
    b = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    s = rng.uniform(0, 1, n).astype(np.float32)
    if ties:
        s = np.round(s * 8).astype(np.float32) / 8
        k = n // 4
        b[-k:] = b[:k]                         # duplicate boxes
        s[-k:] = s[:k]                         # with duplicate scores
    return b, s


@pytest.mark.parametrize("method", ["naive", "linear", "gaussian"])
@pytest.mark.parametrize("n,ties,seed", [(7, False, 0), (60, True, 1), (300, True, 2), (900, False, 3), (2000, True, 4)])
def test_vectorised_restatement_equals_the_literal_loop(method, n, ties, seed):
    if n == 2000 and method != "linear":
        pytest.skip("one literal run at n = 2000 is enough")
    b, s = _random_problem(np.random.default_rng(seed), n, ties)
    _both(b, s, iou_threshold=0.3, sigma=0.5, min_score=0.05 if ties else 1e-3, method=method)


def test_removal_rule_on_its_own():
    rng = np.random.default_rng(7)
    for _ in range(200):
        k = int(rng.integers(1, 30))
        dead = rng.uniform(size=k) < 0.4
        # the literal removal loop over flags
        pos, n, arr = 0, k, list(range(k))
        flags = list(dead)
        while pos < n:
            if flags[pos]:
                arr[pos], flags[pos] = arr[n - 1], flags[n - 1]
                n -= 1
                pos -= 1
            pos += 1
        assert R.removal_order(0, dead).tolist() == arr[:n]


def test_early_exit_is_a_prefix():
    b, s = _random_problem(np.random.default_rng(11), 400, True)
    d, i = R.soft_nms(b, s, min_score=0.05)
    d5, i5 = R.soft_nms(b, s, min_score=0.05, max_keep=5)
    assert np.array_equal(i[:5], i5) and np.array_equal(d[:5], d5)


# ------------------------------------------------------------------------------ config parsing
def test_nms_config_parsing():
    from rsprompter_b200.anchor_heads import parse_nms_cfg
    assert parse_nms_cfg(dict(type="nms", iou_threshold=0.7)) == dict(type="nms", iou_threshold=0.7)
    assert parse_nms_cfg(dict(type="soft_nms", iou_threshold=0.5, min_score=0.05)) == dict(
        type="soft_nms", iou_threshold=0.5, sigma=0.5, min_score=0.05, method="linear")
    assert parse_nms_cfg(dict(type="soft_nms"))["iou_threshold"] == 0.3           # mmcv soft_nms default
    assert parse_nms_cfg(dict(type="nms", iou_threshold=0.5, offset=0, split_thr=10000, class_agnostic=False))
    for bad, word in [(dict(type="nms_match", iou_threshold=0.5), "nms_match"),
                      (dict(type="nms", iou_threshold=0.5, class_agnostic=True), "class_agnostic"),
                      (dict(type="nms", iou_threshold=0.5, offset=1), "offset"),
                      (dict(type="soft_nms", iou_threshold=0.5, split_thr=2000), "split_thr"),
                      (dict(type="nms", iou_threshold=0.5, sigma=0.5), "sigma"),
                      (dict(type="soft_nms", method="matrix"), "matrix"),
                      (dict(type="soft_nms", method="gaussian", sigma=0.0), "sigma")]:
        with pytest.raises(ValueError, match=word):
            parse_nms_cfg(bad)


def _ref_model(name):
    cfg = torch.load(os.path.join(ROOT, "tests", "golden", "reference_configs.pt"), weights_only=False)[name]["model"]
    cfg = copy.deepcopy(cfg)

    def strip(c):
        if isinstance(c, dict):
            c.pop("init_cfg", None)
            for v in c.values():
                strip(v)
        elif isinstance(c, (list, tuple)):
            for v in c:
                strip(v)
    strip(cfg)
    return cfg


@pytest.mark.parametrize("name", ["rsprompter_anchor-nwpu.py", "samseg-maskrcnn-nwpu.py"])
@pytest.mark.parametrize("stage", [None, "rpn", "rcnn"])
def test_reference_configs_build_with_soft_nms(name, stage):
    from rsprompter_b200.registry import MODELS
    cfg = _ref_model(name)
    if stage is not None:
        cfg["test_cfg"][stage]["nms"] = dict(type="soft_nms", iou_threshold=0.5, min_score=0.05)
    m = MODELS.build(cfg)
    assert m.rpn_head._nms["type"] == ("soft_nms" if stage == "rpn" else "nms")
    assert m.roi_head._nms["type"] == ("soft_nms" if stage == "rcnn" else "nms")
    cfg["test_cfg"]["rcnn"]["nms"] = dict(type="soft_nms", iou_threshold=0.5, nms_match=True)
    with pytest.raises(ValueError, match="nms_match"):
        MODELS.build(cfg)


# ------------------------------------------------------------------------------ ptxas
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")


def test_soft_nms_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "detect.ptxas.log")) as f:
        log = f.read()
    spills, cur = {}, None
    for line in log.splitlines():
        m = ENTRY.search(line)
        if m:
            cur = m.group(1)
            continue
        m = SPILLS.search(line)
        if m and cur is not None and "soft_nms" in cur:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(spills) == 3, sorted(spills)
    assert all(v == (0, 0) for v in spills.values()), spills
