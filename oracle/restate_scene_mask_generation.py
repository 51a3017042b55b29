"""Plain-torch restatement of segment-everything over a whole scene (TEST INFRASTRUCTURE, see oracle/__init__.py):
restate_mask_generation's pipeline per window, with HF's crop-edge rule where filter_masks applies it (after the
predicted-IoU and stability filters, before the window's NMS), optionally SAM's small-region step, then the shift into
scene coordinates and one box NMS over every window's survivors.  rsprompter_b200.mask_generation.generate_scene_masks
is checked against it; tests/test_scene_mask_generation_cpu.py pins the rule and the uncrop to transformers' own
_is_box_near_crop_edge and _pad_masks.

Citations: P: = transformers/models/sam/image_processing_sam.py (transformers 5.5.0)."""
from __future__ import annotations

import torch

from . import restate_large_image as L
from . import restate_mask_generation as R
from . import restate_small_regions as S

EDGE_ATOL = 20.0         # filter_masks' _is_box_near_crop_edge(..., atol=20) default (P:509)


def crop_boxes(hw: tuple, patch: int, overlap_ratio: float) -> list:
    """The windows of a scene as crop boxes: sahi's slice origins (restate_large_image.slice_origins), each window cut
    to its in-scene part, (x0, y0, min(x0 + P, W), min(y0 + P, H))."""
    H, W = hw
    return [(x0, y0, min(x0 + patch, W), min(y0 + patch, H)) for x0, y0 in L.slice_origins(hw, patch, overlap_ratio)]


def near_crop_edge(boxes: torch.Tensor, crop_box, scene_hw, atol: float = EDGE_ATOL) -> torch.Tensor:
    """_is_box_near_crop_edge(boxes, crop_box, [0, 0, W, H], atol) (P:509-525) for inclusive xyxy boxes in crop
    pixels: shifted by the crop's origin and rounded to fp32, a side is near when |side - crop side| <= atol and not
    |side - scene side| <= atol.  -> bool [n]."""
    H, W = scene_hw
    x0, y0 = crop_box[0], crop_box[1]
    b = (boxes.long() + torch.tensor([[x0, y0, x0, y0]])).float()
    crop = torch.tensor([list(crop_box)], dtype=torch.float32)
    scene = torch.tensor([[0, 0, W, H]], dtype=torch.float32)
    return (((b - crop).abs() <= atol) & ~((b - scene).abs() <= atol)).any(1)


def uncrop(masks: torch.Tensor, crop_box, scene_hw) -> torch.Tensor:
    """The masks [k, h, w] of a crop as masks of the whole scene [k, H, W] (what _pad_masks, P:527-534, does)."""
    H, W = scene_hw
    x0, y0, x1, y1 = crop_box
    out = torch.zeros(masks.shape[0], H, W, dtype=masks.dtype)
    out[:, y0:y1, x0:x1] = masks
    return out


def generate_window(low_res: torch.Tensor, iou_scores: torch.Tensor, crop_box, scene_hw, reshaped_size: tuple,
                    pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95,
                    stability_score_offset: float = 1.0, mask_threshold: float = 0.0, crops_nms_thresh: float = 0.7,
                    min_mask_region_area: float = 0.0, pad_size=(1024, 1024)) -> dict:
    """restate_mask_generation.generate for the window crop_box of the scene, with the crop-edge rule added to the
    filters' keep mask before the NMS, then restate_small_regions' step when min_mask_region_area > 0.
    -> dict(index, scores, stability, boxes (crop pixels), masks bool [k, h, w]), rows in the window's final order."""
    x0, y0, x1, y1 = crop_box
    hw = (y1 - y0, x1 - x0)
    masks = R.upscale(low_res, hw, reshaped_size, pad_size).flatten(0, 1)
    iou = iou_scores.flatten(0, 1).float()
    st = R.mask_stats(masks, mask_threshold, stability_score_offset)
    keep = torch.ones(len(iou), dtype=torch.bool)
    if pred_iou_thresh > 0.0:
        keep &= iou > pred_iou_thresh
    if stability_score_thresh > 0.0:
        keep &= st["stability"] > stability_score_thresh
    keep &= ~near_crop_edge(st["boxes"], crop_box, scene_hw)
    cand = torch.nonzero(keep).view(-1)
    index = cand[R.nms(st["boxes"][cand], iou[cand], crops_nms_thresh)]
    out = dict(index=index, scores=iou[index], stability=st["stability"][index], boxes=st["boxes"][index],
               masks=st["binary"][index])
    if min_mask_region_area > 0:
        pp = S.postprocess_small_regions(out["masks"], min_mask_region_area, crops_nms_thresh)
        rows = pp["index"]
        out = dict(index=index[rows], scores=out["scores"][rows], stability=out["stability"][rows], boxes=pp["boxes"],
                   masks=pp["masks"])
    return out


def merge(windows: list, crops: list, points: list, crops_nms_thresh: float) -> dict:
    """The cross-window merge: every window's rows (``windows[t]`` from generate_window, ``points[t]`` the window's
    prompts fp32 [n_points, 2] in window pixels) shifted into the scene (integer boxes, fp32 points) and de-duplicated
    by one box NMS scored by predicted IoU; the stable sort breaks ties by (window, rank in the window).
    -> dict(tiles, candidates, scores, stability, boxes, points, rank), rows in keep order; ``rank`` is the row's
    position in its window's result."""
    tiles, ranks, boxes, pts = [], [], [], []
    for t, (w, cb) in enumerate(zip(windows, crops)):
        k = len(w["index"])
        tiles.append(torch.full((k,), t, dtype=torch.int64))
        ranks.append(torch.arange(k))
        boxes.append(w["boxes"].long() + torch.tensor([[cb[0], cb[1], cb[0], cb[1]]]))
        pts.append(points[t][w["index"] // 3] + torch.tensor([[cb[0], cb[1]]], dtype=torch.float32))
    tiles, ranks, boxes, pts = torch.cat(tiles), torch.cat(ranks), torch.cat(boxes), torch.cat(pts)
    cands = torch.cat([w["index"] for w in windows])
    scores = torch.cat([w["scores"] for w in windows])
    stab = torch.cat([w["stability"] for w in windows])
    keep = R.nms(boxes, scores, crops_nms_thresh)
    return dict(tiles=tiles[keep], candidates=cands[keep], scores=scores[keep], stability=stab[keep],
                boxes=boxes[keep], points=pts[keep], rank=ranks[keep])
