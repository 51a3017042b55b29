"""Restatement of SAM's small-region removal (TEST INFRASTRUCTURE ONLY): ``remove_small_regions``
(segment_anything/utils/amg.py) and ``SamAutomaticMaskGenerator.postprocess_small_regions``
(segment_anything/automatic_mask_generator.py), the ``min_mask_region_area`` step of SAM's automatic mask generator.

``segment_anything`` is not installed here: both functions are restated from SAM's published code, on top of the same
``cv2.connectedComponentsWithStats(working_mask, 8)`` they call, so the component analysis is cv2's own.  The
hand-worked cases of tests/test_small_regions_cpu.py pin the restatement.  One deliberate difference: the second NMS
uses ``restate_mask_generation.nms``, whose sort is stable (ties keep the first NMS's order); SAM's torchvision
``batched_nms`` sorts without that guarantee.

``generate`` composes it with ``restate_mask_generation.generate``: the reference of ``generate_masks(...,
min_mask_region_area=A)``."""
from __future__ import annotations

import math

import cv2
import numpy as np
import torch

from . import restate_mask_generation as R


def remove_small_regions(mask: np.ndarray, area_thresh: float, mode: str) -> tuple:
    """amg.py remove_small_regions: mask bool [H, W] -> (mask bool [H, W], changed).  "holes" fills background
    components of area < area_thresh (border ones included); "islands" keeps the foreground components of area >=
    area_thresh, or only the largest (first cv2 label on ties) when there are none.  changed = some component is
    small, whether or not the mask then differs."""
    assert mode in ("holes", "islands")
    correct_holes = mode == "holes"
    working_mask = (correct_holes ^ mask).astype(np.uint8)
    n_labels, regions, stats, _ = cv2.connectedComponentsWithStats(working_mask, 8)
    sizes = stats[:, -1][1:]                                       # row 0 is the background label
    small_regions = [i + 1 for i, s in enumerate(sizes) if s < area_thresh]
    if len(small_regions) == 0:
        return mask, False
    fill_labels = [0] + small_regions
    if not correct_holes:
        fill_labels = [i for i in range(n_labels) if i not in fill_labels]
        if len(fill_labels) == 0:                                  # every region is small: keep the largest
            fill_labels = [int(np.argmax(sizes)) + 1]
    return np.isin(regions, fill_labels), True


def mask_to_box(masks: torch.Tensor) -> torch.Tensor:
    """batched_mask_to_box (amg.py) = HF's _batched_mask_to_box: bool [k, H, W] -> inclusive xyxy int64 [k, 4],
    zeros for an empty mask."""
    return R.mask_stats(masks.float(), 0.5, 0.0)["boxes"]


def postprocess_small_regions(masks: torch.Tensor, min_area: float, nms_thresh: float) -> dict:
    """postprocess_small_regions on the kept masks bool [k, H, W] (in the first NMS's keep order): holes then islands
    per mask, score = float(unchanged), boxes of the cleaned masks, a box NMS at nms_thresh.
    -> dict(index = rows of ``masks`` in the new keep order, masks = cleaned masks of those rows, boxes, changed
    bool [k] of every row)."""
    k = masks.shape[0]
    if k == 0:
        return dict(index=torch.zeros(0, dtype=torch.int64), masks=masks, boxes=torch.zeros(0, 4, dtype=torch.int64),
                    changed=torch.zeros(0, dtype=torch.bool))
    new_masks, scores = [], []
    for m in masks.numpy():
        m, changed = remove_small_regions(m, min_area, "holes")
        unchanged = not changed
        m, changed = remove_small_regions(m, min_area, "islands")
        unchanged = unchanged and not changed
        new_masks.append(torch.as_tensor(m))
        scores.append(float(unchanged))
    cleaned = torch.stack(new_masks)
    boxes = mask_to_box(cleaned)
    keep = R.nms(boxes, torch.tensor(scores), nms_thresh)
    return dict(index=keep, masks=cleaned[keep], boxes=boxes[keep], changed=torch.tensor(scores) == 0.0)


def generate(low_res: torch.Tensor, iou_scores: torch.Tensor, original_size: tuple, reshaped_size: tuple,
             min_mask_region_area: float, crops_nms_thresh: float = 0.7, **kw) -> dict:
    """restate_mask_generation.generate followed, when min_mask_region_area > 0, by postprocess_small_regions at
    crops_nms_thresh.  -> the same keys as generate (index, scores, stability, boxes, masks), rows in the final order."""
    ref = R.generate(low_res, iou_scores, original_size, reshaped_size, crops_nms_thresh=crops_nms_thresh, **kw)
    if not min_mask_region_area > 0:
        return ref
    assert math.isfinite(min_mask_region_area)
    pp = postprocess_small_regions(ref["masks"], min_mask_region_area, crops_nms_thresh)
    rows = pp["index"]
    out = dict(ref, index=ref["index"][rows], scores=ref["scores"][rows], stability=ref["stability"][rows],
               boxes=pp["boxes"], masks=pp["masks"], after_small_regions=len(rows), changed=pp["changed"])
    return out
