"""Restatement of the reference's large-image inference (TEST INFRASTRUCTURE ONLY): demo/large_image_demo.py:141-262
slices the scene with sahi, runs every slice, and merges with mmdet/utils/large_image.py:27-104
(``shift_predictions`` + ``merge_results_by_nms``).

sahi is neither a dependency of the reference tree nor installed here.  ``slice_origins`` (sahi.slicing
get_slice_bboxes, as ``slice_image(..., auto_slice_resolution=False)`` calls it) and ``shift_masks`` (paste into a
full-scene bool canvas) are restated from memory; the worked examples of tests/test_large_image_cpu.py pin them.
``shift_bboxes`` is the fp32 add ``bboxes + offset``.  mmcv ``batched_nms`` is ``restate_anchor.batched_nms``."""
from __future__ import annotations

import torch

from .restate_anchor import batched_nms


def slice_origins(hw, patch: int, overlap_ratio: float) -> list:
    """sahi get_slice_bboxes(image_height=H, image_width=W, slice_height=slice_width=patch, overlap ratios equal):
    the (x_min, y_min) of every slice, row-major; edge slices are shifted inward."""
    H, W = hw
    ov = int(overlap_ratio * patch)
    boxes = []
    y_min = y_max = 0
    while y_max < H:
        x_min = x_max = 0
        y_max = y_min + patch
        while x_max < W:
            x_max = x_min + patch
            if y_max > H or x_max > W:
                xmax, ymax = min(W, x_max), min(H, y_max)
                boxes.append((max(0, xmax - patch), max(0, ymax - patch)))
            else:
                boxes.append((x_min, y_min))
            x_min = x_max - ov
        y_min = y_max - ov
    return boxes


def shift_masks(masks: torch.Tensor, offset, src_hw) -> torch.Tensor:
    """sahi shift_masks: every mask pasted at its slice's offset into an all-False scene canvas (the part of the mask
    that falls outside the scene is dropped)."""
    H, W = src_hw
    x0, y0 = offset
    out = torch.zeros(masks.shape[0], H, W, dtype=torch.bool)
    h, w = min(masks.shape[1], H - y0), min(masks.shape[2], W - x0)
    out[:, y0:y0 + h, x0:x0 + w] = masks[:, :h, :w].bool()
    return out


def shift_predictions(tiles: list, offsets: list, src_hw, patch: int | None = None) -> dict:
    """large_image.py:27-73: per-tile dict(bboxes [n, 4], scores, labels[, masks [n, h, w]]) -> one dict in scene
    coordinates, tiles concatenated in order (InstanceData.cat).  With ``patch``, each shifted box is also clipped to
    its tile's window intersected with the scene: this package pads a tile that overhangs a scene smaller than the
    patch, and a box can reach into that padding.  For a box inside its tile the clip is a no-op."""
    H, W = src_hw
    out = dict(bboxes=[], scores=[], labels=[], masks=[])
    for t, (x0, y0) in zip(tiles, offsets):
        b = t["bboxes"].float() + torch.tensor([x0, y0, x0, y0], dtype=torch.float32)
        if patch is not None:
            lo = torch.tensor([x0, y0, x0, y0], dtype=torch.float32)
            hi = torch.tensor([min(x0 + patch, W), min(y0 + patch, H)] * 2, dtype=torch.float32)
            b = torch.minimum(torch.maximum(b, lo), hi)
        out["bboxes"].append(b)
        out["scores"].append(t["scores"].float())
        out["labels"].append(t["labels"].long())
        if "masks" in t:
            out["masks"].append(shift_masks(t["masks"], (x0, y0), src_hw))
    res = {k: torch.cat(v) for k, v in out.items() if v}
    res.setdefault("bboxes", torch.zeros(0, 4))
    return res


def merge_results_by_nms(tiles: list, offsets: list, src_hw, iou_thr: float, patch: int | None = None):
    """large_image.py:76-104 with nms_cfg = dict(type='nms', iou_threshold=iou_thr) -> (merged dict in descending
    score order, keep = indices into the concatenated tiles)."""
    inst = shift_predictions(tiles, offsets, src_hw, patch)
    if inst["bboxes"].shape[0] == 0:
        return inst, torch.zeros(0, dtype=torch.long)
    _, keep = batched_nms(inst["bboxes"], inst["scores"], inst["labels"], iou_thr)
    return {k: v[keep] for k, v in inst.items()}, keep
