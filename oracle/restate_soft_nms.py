"""Restatement of mmcv's soft-NMS (TEST INFRASTRUCTURE ONLY): ``mmcv.ops.soft_nms`` / ``softnms_cpu``
(mmcv/ops/csrc/pytorch/cpu/nms.cpp) and the ``type='soft_nms'`` branch of ``mmcv.ops.batched_nms``, mmcv 2.1.0.

mmcv is neither a dependency of the reference tree nor installed here: the loop below is restated FROM MEMORY, and the
hand-worked examples of tests/test_soft_nms_cpu.py pin it.  The comparisons whose direction matters are the three
``_SELECT`` / ``_DECAY`` / ``_REMOVE`` predicates, kept in one place so that they can be checked against the mmcv
source.  Arithmetic is fp32 in softnms_cpu's order, with no fused multiply-add.  The gaussian weight is
``exp`` in float64 of the fp32 argument, rounded once to fp32; mmcv's ``std::exp(float)`` may differ from that by an
ulp.

``soft_nms_literal`` is the serial loop, statement for statement.  ``soft_nms`` is the same algorithm vectorised per
step with numpy, for problems of thousands of candidates; it relies on the removal rule below, which the CPU tests pin
against the literal loop.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .restate_anchor import batched_nms as _hard_batched_nms

METHODS = {"naive": 0, "linear": 1, "gaussian": 2}
SPLIT_THR = 10000


def _SELECT(max_score, s) -> bool:          # the running max is replaced only by a strictly greater score
    return max_score < s


def _DECAY(ovr, thr) -> bool:               # naive / linear act at ovr >= iou_threshold (the paper uses >)
    return ovr >= thr


def _REMOVE(s, min_score) -> bool:          # dropped when below min_score
    return s < min_score


def _f32(x) -> np.float32:
    return np.float32(x)


def _weight(ovr: np.float32, thr: np.float32, sigma: np.float32, method: int) -> np.float32:
    if method == 0:
        return _f32(0.0) if _DECAY(ovr, thr) else _f32(1.0)
    if method == 1:
        return _f32(_f32(1.0) - ovr) if _DECAY(ovr, thr) else _f32(1.0)
    arg = _f32(_f32(-(ovr * ovr)) / sigma)
    return _f32(math.exp(float(arg))) if not math.isnan(arg) else _f32("nan")


def soft_nms_literal(boxes, scores, iou_threshold=0.3, sigma=0.5, min_score=1e-3, method="linear", offset=0):
    """softnms_cpu, line for line.  boxes fp32 [n, 4], scores fp32 [n] -> (dets fp32 [k, 5] = box + decayed score,
    inds int64 [k]) in selection order."""
    method = METHODS[method]
    b = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    x1, y1, x2, y2 = (list(b[:, c]) for c in range(4))
    sc = list(np.asarray(scores, dtype=np.float32).reshape(-1))
    off = _f32(offset)
    areas = [_f32(_f32(_f32(x2[k] - x1[k]) + off) * _f32(_f32(y2[k] - y1[k]) + off)) for k in range(len(sc))]
    inds = list(range(len(sc)))
    thr, sig, mins = _f32(iou_threshold), _f32(sigma), _f32(min_score)
    n = len(sc)
    dets = []
    i = 0
    while i < n:
        max_score, max_pos = sc[i], i
        pos = i + 1
        while pos < n:
            if _SELECT(max_score, sc[pos]):
                max_score, max_pos = sc[pos], pos
            pos += 1
        for arr in (x1, y1, x2, y2, sc, areas, inds):
            arr[i], arr[max_pos] = arr[max_pos], arr[i]
        ix1, iy1, ix2, iy2, iarea = x1[i], y1[i], x2[i], y2[i], areas[i]
        dets.append((ix1, iy1, ix2, iy2, sc[i]))
        pos = i + 1
        while pos < n:
            xx1, yy1 = max(ix1, x1[pos]), max(iy1, y1[pos])
            xx2, yy2 = min(ix2, x2[pos]), min(iy2, y2[pos])
            w = max(_f32(0.0), _f32(_f32(xx2 - xx1) + off))
            h = max(_f32(0.0), _f32(_f32(yy2 - yy1) + off))
            inter = _f32(w * h)
            with np.errstate(invalid="ignore", divide="ignore"):
                ovr = _f32(inter / _f32(_f32(iarea + areas[pos]) - inter))
            sc[pos] = _f32(sc[pos] * _weight(ovr, thr, sig, method))
            if _REMOVE(sc[pos], mins):
                for arr in (x1, y1, x2, y2, sc, areas, inds):
                    arr[pos] = arr[n - 1]
                n -= 1
                pos -= 1
            pos += 1
        i += 1
    d = np.array(dets, dtype=np.float32).reshape(-1, 5)
    return d[:n], np.array(inds[:n], dtype=np.int64)


def removal_order(n_front: int, dead: np.ndarray) -> np.ndarray:
    """Positions after one step's removal.  ``dead`` flags positions i+1 .. n-1 (already decayed): the m survivors end
    at i+1+m; survivors below that end stay, and each removed slot below it is filled by a survivor from above it,
    lowest slot first, highest survivor first.  Returns the old relative positions of the new ones."""
    m = int((~dead).sum())
    rel = np.arange(dead.shape[0])
    out = rel[:m].copy()
    holes = np.nonzero(dead[:m])[0]
    tail = rel[m:][~dead[m:]][::-1]
    out[holes] = tail
    return out


def soft_nms(boxes, scores, iou_threshold=0.3, sigma=0.5, min_score=1e-3, method="linear", offset=0, max_keep=0):
    """soft_nms_literal vectorised per step (same fp32 operations, elementwise).  max_keep > 0 stops after that many
    selections, which are final once made."""
    method = METHODS[method]
    b = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    x1, y1, x2, y2 = (b[:, c].copy() for c in range(4))
    sc = np.asarray(scores, dtype=np.float32).reshape(-1).copy()
    off = _f32(offset)
    area = ((x2 - x1) + off) * ((y2 - y1) + off)
    inds = np.arange(sc.shape[0], dtype=np.int64)
    thr, sig, mins = _f32(iou_threshold), _f32(sigma), _f32(min_score)
    n = sc.shape[0]
    dets = []
    i = 0
    stop = n if max_keep <= 0 else max_keep
    while i < n and i < stop:
        seg = sc[i:n]
        if np.isnan(seg[0]):
            p = i
        else:
            with np.errstate(invalid="ignore"):
                finite = np.where(np.isnan(seg), -np.inf, seg)
            p = i + int(np.argmax(finite))          # first position of the largest score
        for arr in (x1, y1, x2, y2, sc, area, inds):
            arr[i], arr[p] = arr[p], arr[i]
        dets.append((x1[i], y1[i], x2[i], y2[i], sc[i]))
        lo = i + 1
        if lo < n:
            s = slice(lo, n)
            w = np.maximum(_f32(0.0), (np.minimum(x2[i], x2[s]) - np.maximum(x1[i], x1[s])) + off)
            h = np.maximum(_f32(0.0), (np.minimum(y2[i], y2[s]) - np.maximum(y1[i], y1[s])) + off)
            inter = w * h
            with np.errstate(invalid="ignore", divide="ignore"):
                ovr = inter / ((area[i] + area[s]) - inter)
                if method == 0:
                    wt = np.where(_DECAY(ovr, thr), _f32(0.0), _f32(1.0)).astype(np.float32)
                elif method == 1:
                    wt = np.where(_DECAY(ovr, thr), _f32(1.0) - ovr, _f32(1.0)).astype(np.float32)
                else:
                    arg = (-(ovr * ovr)) / sig
                    wt = np.exp(arg.astype(np.float64)).astype(np.float32)
                sc[s] = sc[s] * wt
                dead = _REMOVE(sc[s], mins)
            if dead.any():
                order = lo + removal_order(lo, dead)
                for arr in (x1, y1, x2, y2, sc, area, inds):
                    arr[lo:lo + order.shape[0]] = arr[order]
                n = lo + order.shape[0]
        i += 1
    d = np.array(dets, dtype=np.float32).reshape(-1, 5)
    return d, inds[:i].copy()


def batched_nms(boxes: torch.Tensor, scores: torch.Tensor, idxs: torch.Tensor, nms_cfg, split_thr: int = SPLIT_THR,
                max_keep: int = 0):
    """mmcv.ops.batched_nms(boxes, scores, idxs, nms_cfg) for type 'nms' (restate_anchor.batched_nms; a float is read
    as iou_threshold) and 'soft_nms'.  Boxes are offset by idx * (max + 1); below split_thr one soft_nms in input
    order, output in selection order; otherwise one per idx, then an unstable sort by decayed score (here: stable, ties
    by idx then selection order).  Returns (dets [k, 5] with the un-offset boxes and the decayed scores, keep).
    max_keep > 0 (soft, below split_thr only): the first max_keep selections."""
    cfg = dict(type="nms", iou_threshold=nms_cfg) if isinstance(nms_cfg, (int, float)) else dict(nms_cfg)
    typ = cfg.pop("type", "nms")
    if typ == "nms":
        return _hard_batched_nms(boxes, scores, idxs, cfg["iou_threshold"], split_thr)
    assert typ == "soft_nms", typ
    kw = dict(iou_threshold=cfg.get("iou_threshold", 0.3), sigma=cfg.get("sigma", 0.5),
              min_score=cfg.get("min_score", 1e-3), method=cfg.get("method", "linear"))
    if boxes.numel() == 0:
        return torch.cat([boxes, scores[:, None]], -1), boxes.new_zeros(0, dtype=torch.long)
    boxes, scores = boxes.float(), scores.float()
    mx = boxes.max()
    bfn = boxes + (idxs.to(boxes) * (mx + boxes.new_tensor(1)))[:, None]
    if bfn.shape[0] < split_thr:
        d, keep = soft_nms(bfn.numpy(), scores.numpy(), max_keep=max_keep, **kw)
        keep = torch.from_numpy(keep)
        return torch.cat([boxes[keep], torch.from_numpy(d[:, 4])[:, None]], -1), keep
    rows = []
    for c in torch.unique(idxs).tolist():
        m = (idxs == c).nonzero(as_tuple=False).view(-1)
        d, k = soft_nms(bfn[m].numpy(), scores[m].numpy(), **kw)
        rows += [(-float(s), c, j, int(m[kk])) for j, (s, kk) in enumerate(zip(d[:, 4], k))]
    rows.sort()
    keep = torch.tensor([r[3] for r in rows], dtype=torch.long)
    s = torch.tensor([-r[0] for r in rows], dtype=torch.float32)
    return torch.cat([boxes[keep], s[:, None]], -1), keep


def multiclass_nms(bboxes: torch.Tensor, scores: torch.Tensor, score_thr: float, nms_cfg, max_num: int = -1):
    """mmdet multiclass_nms (bbox_nms.py:13-105) for per-class boxes: bboxes [n, C*4], scores [n, C+1] (softmax,
    background last).  Candidates are the (row, class) pairs with score > score_thr, row-major.  -> (dets [k, 5],
    labels [k])."""
    C = scores.shape[1] - 1
    b = bboxes.reshape(-1, C, 4).reshape(-1, 4)
    s = scores[:, :-1].reshape(-1)
    labels = torch.arange(C).view(1, -1).expand(scores.shape[0], C).reshape(-1)
    inds = (s > score_thr).nonzero(as_tuple=False).squeeze(1)
    b, s, labels = b[inds], s[inds], labels[inds]
    if b.numel() == 0:
        return b.new_zeros(0, 5), labels
    dets, keep = batched_nms(b, s, labels, nms_cfg)
    if max_num > 0:
        dets, keep = dets[:max_num], keep[:max_num]
    return dets, labels[keep]


def bbox_predict_single(roi, cls_score, bbox_pred, img_shape, num_classes: int, nms_cfg, score_thr=0.05,
                        max_per_img=100, stds=(0.1, 0.1, 0.2, 0.2)):
    """BBoxHead._predict_by_feat_single + multiclass_nms (bbox_head.py:476-571) with any nms_cfg.
    -> (bboxes [k, 4], scores [k], labels [k])."""
    from .restate_anchor import delta2bbox
    sm = torch.softmax(cls_score, dim=-1)
    n = roi.size(0)
    r = roi.repeat_interleave(num_classes, dim=0)
    boxes = delta2bbox(r[:, 1:], bbox_pred.reshape(-1, 4), stds, img_shape).view(n, -1)
    dets, labels = multiclass_nms(boxes, sm, score_thr, nms_cfg, max_per_img)
    return dets[:, :4], dets[:, 4], labels


def rpn_nms(boxes: torch.Tensor, scores: torch.Tensor, level_ids: torch.Tensor, nms_cfg, max_per_img: int):
    """RPNHead._bbox_post_process's NMS (rpn_head.py:285-291) on the per-level top-k candidates in level order:
    results[keep] with scores = the decayed ones, then [:max_per_img].  -> (boxes, scores)."""
    if boxes.numel() == 0:
        return boxes.new_zeros(0, 4), scores.new_zeros(0)
    dets, keep = batched_nms(boxes.float(), scores.float(), level_ids, nms_cfg)
    return boxes[keep][:max_per_img], dets[:, -1][:max_per_img]


def merge_results_by_nms(tiles: list, offsets: list, src_hw, nms_cfg, patch: int | None = None):
    """mmdet/utils/large_image.py:76-104 with any nms_cfg: ``_, keeps = batched_nms(...)`` then
    ``shifted_instances[keeps]``, so the kept rows carry their original scores, in keep order.
    -> (merged dict, keep)."""
    from .restate_large_image import shift_predictions
    inst = shift_predictions(tiles, offsets, src_hw, patch)
    if inst["bboxes"].shape[0] == 0:
        return inst, torch.zeros(0, dtype=torch.long)
    _, keep = batched_nms(inst["bboxes"], inst["scores"], inst["labels"], nms_cfg)
    return {k: v[keep] for k, v in inst.items()}, keep
