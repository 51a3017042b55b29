"""Greedy non-maximum merging of tiled detections (TEST INFRASTRUCTURE ONLY), the semantics of
rsprompter_b200.large_image.merge_tile_records(..., nms_type='greedy_nmm').

It follows sahi's GREEDYNMM postprocess (greedy_nmm grouping, then a merge of each group) as it is commonly
described; sahi is not installed here and nothing is taken from its code.  The semantics are pinned by the worked
examples of tests/test_nmm_cpu.py, not by a claim of equality with any sahi version.  One deliberate difference:
sahi's loop tests each member again against the growing merged box and drops it when it no longer matches; here every
matched member joins its group.

  * candidates: every tile's rows shifted into the scene (restate_large_image.shift_predictions, clipped to the tile
    window with ``patch``), those below ``score_thr`` dropped, sorted by score, descending, ties by (tile, slot);
  * match(i, j): equal labels and metric >= thr, in fp32 with every step rounded: area = (x2 - x1) * (y2 - y1),
    inter = max(0, min(x2) - max(x1)) * max(0, min(y2) - max(y1)), iou = inter / ((area_i + area_j) - inter),
    ios = inter / min(area_i, area_j); a NaN does not match;
  * greedy: in sort order, a candidate no keeper absorbed is a keeper and absorbs every later unabsorbed candidate
    it matches;
  * a keeper's row: the element-wise min of x1, y1 and max of x2, y2 over its group, its own score and label, and the
    OR of its group's scene masks (shift_masks)."""
from __future__ import annotations

import torch

from .restate_large_image import shift_masks, shift_predictions


def match(a: torch.Tensor, b: torch.Tensor, metric: str, thr: float) -> torch.Tensor:
    """a fp32 [4], b fp32 [n, 4] -> bool [n]: metric(a, b[j]) >= thr (labels are compared by the caller)."""
    w = torch.clamp(torch.minimum(a[2], b[:, 2]) - torch.maximum(a[0], b[:, 0]), min=0)
    h = torch.clamp(torch.minimum(a[3], b[:, 3]) - torch.maximum(a[1], b[:, 1]), min=0)
    inter = w * h
    sa = (a[2] - a[0]) * (a[3] - a[1])
    sb = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    if metric == "iou":
        v = inter / ((sa + sb) - inter)
    elif metric == "ios":
        v = inter / torch.minimum(sa.expand_as(sb), sb)
    else:
        raise ValueError(metric)
    return v >= torch.tensor(thr, dtype=torch.float32)          # NaN >= thr is False


def greedy_nmm(boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, thr: float, metric: str = "ios"):
    """Candidates in input order (ties by that order) -> groups: a list of index lists into the input, one per keeper
    in descending score order, each its keeper first, then its absorbed members in sort order."""
    order = torch.sort(scores.float(), descending=True, stable=True)[1]
    b, lab = boxes.float()[order], labels.long()[order]                 # in sort order
    n = int(order.numel())
    absorbed = torch.zeros(n, dtype=torch.bool)
    groups = []
    for p in range(n):
        if absorbed[p]:
            continue
        # every later candidate at once: the unabsorbed ones that match keeper p join it
        hit = ~absorbed[p + 1:] & (lab[p + 1:] == lab[p]) & match(b[p], b[p + 1:], metric, thr)
        absorbed[p + 1:] |= hit
        groups.append([p] + (torch.nonzero(hit).view(-1) + p + 1).tolist())
    return [order[g].tolist() for g in groups]


def merge_groups(boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor, groups: list) -> dict:
    """The merged rows of greedy_nmm's groups: union box, keeper score and label."""
    if not groups:
        return dict(bboxes=torch.zeros(0, 4), scores=torch.zeros(0), labels=torch.zeros(0, dtype=torch.long))
    out = []
    for g in groups:
        b = boxes[g].float()
        out.append(torch.cat([b[:, :2].min(0).values, b[:, 2:].max(0).values]))
    keepers = torch.tensor([g[0] for g in groups])
    return dict(bboxes=torch.stack(out), scores=scores[keepers].float(), labels=labels[keepers].long())


def merge_results_by_nmm(tiles: list, offsets: list, src_hw, thr: float, metric: str = "ios",
                         patch: int | None = None, score_thr: float = 0.0):
    """Per-tile dict(bboxes, scores, labels) -> (merged dict, groups as index lists into the concatenated tiles)."""
    inst = shift_predictions(tiles, offsets, src_hw, patch)
    n = inst["bboxes"].shape[0]
    if n == 0:
        return merge_groups(inst["bboxes"], torch.zeros(0), torch.zeros(0, dtype=torch.long), []), []
    cand = torch.nonzero(inst["scores"] >= score_thr).view(-1) if score_thr > 0 else torch.arange(n)
    groups = greedy_nmm(inst["bboxes"][cand], inst["scores"][cand], inst["labels"][cand], thr, metric)
    groups = [[int(cand[j]) for j in g] for g in groups]
    return merge_groups(inst["bboxes"], inst["scores"], inst["labels"], groups), groups


def union_masks(masks: list, offsets: list, src_hw) -> torch.Tensor:
    """The OR of masks[k] (bool [h, w]) each placed at offsets[k] = (x0, y0) in the scene -> bool [H, W]."""
    out = torch.zeros(int(src_hw[0]), int(src_hw[1]), dtype=torch.bool)
    for m, o in zip(masks, offsets):
        out |= shift_masks(torch.as_tensor(m)[None], o, src_hw)[0]
    return out
