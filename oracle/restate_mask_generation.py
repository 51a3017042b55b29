"""Plain-torch restatement of HF's SAM mask generation for one crop layer (TEST INFRASTRUCTURE, see oracle/__init__.py):
the point grid and its normalisation, post_process_masks(binarize=False), filter_masks and
post_process_for_mask_generation, on decoder outputs given to it.  The kernels of rsprompter_b200.mask_generation are
checked against it, and it is pinned to transformers' own functions by tests/test_mask_generation_cpu.py.

Citations: P: = transformers/models/sam/image_processing_sam.py, G: = transformers/pipelines/mask_generation.py
(transformers 5.5.0)."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def build_point_grid(n_per_side: int) -> torch.Tensor:
    """_build_point_grid (P:624-631): n x n points evenly spaced in [0, 1]^2, x fastest, fp32 [n * n, 2]."""
    offset = 1 / (2 * n_per_side)
    side = torch.linspace(offset, 1 - offset, n_per_side)
    xs = side[None, :].expand(n_per_side, n_per_side)
    ys = side[:, None].expand(n_per_side, n_per_side)
    return torch.stack([xs, ys], dim=-1).reshape(-1, 2)


def normalize_coordinates(target_size: int, coords: torch.Tensor, original_size: tuple) -> torch.Tensor:
    """_normalize_coordinates (P:659-684): original-pixel xy -> the frame of the image resized to longest edge
    target_size (each axis by new / old, new = int(old * scale + 0.5))."""
    old_h, old_w = original_size
    scale = target_size * 1.0 / max(old_h, old_w)
    new_h, new_w = int(old_h * scale + 0.5), int(old_w * scale + 0.5)
    out = coords.float().clone()
    out[..., 0] = out[..., 0] * (new_w / old_w)
    out[..., 1] = out[..., 1] * (new_h / old_h)
    return out


def grid_prompts(n_per_side: int, original_size: tuple, target_size: int = 1024) -> tuple:
    """The whole-image crop of _generate_crop_images (P:643-654): grid * (W, H), then normalised.
    -> (points in original pixels, points in the model frame), fp32 [n * n, 2]."""
    H, W = original_size
    pts = build_point_grid(n_per_side) * torch.tensor([[W, H]])
    return pts, normalize_coordinates(target_size, pts, (H, W))


def upscale(low_res: torch.Tensor, original_size: tuple, reshaped_size: tuple, pad_size=(1024, 1024)) -> torch.Tensor:
    """post_process_masks(binarize=False) (P:423-425): [..., hm, wm] -> bilinear to pad_size, crop to the reshaped
    input size, bilinear to the original size; fp32 [..., H, W]."""
    lead = low_res.shape[:-2]
    x = low_res.reshape(1, -1, *low_res.shape[-2:]).float()
    x = F.interpolate(x, tuple(pad_size), mode="bilinear", align_corners=False)
    x = x[..., :reshaped_size[0], :reshaped_size[1]]
    x = F.interpolate(x, tuple(original_size), mode="bilinear", align_corners=False)
    return x.reshape(*lead, *x.shape[-2:])


def mask_stats(masks: torch.Tensor, mask_threshold: float, offset: float) -> dict:
    """Per mask of fp32 masks [n, H, W]: the counts of _compute_stability_score (P:449-457, summed in int32: HF's
    int16 row sums agree for W < 32768), the stability score as int32 / int32 true division, and _batched_mask_to_box
    (P:460-506) of masks > mask_threshold: inclusive xyxy int64, zeros when empty."""
    hi = (masks > (mask_threshold + offset)).sum((-2, -1), dtype=torch.int32)
    lo = (masks > (mask_threshold - offset)).sum((-2, -1), dtype=torch.int32)
    binary = masks > mask_threshold
    mid = binary.sum((-2, -1), dtype=torch.int32)
    n, H, W = binary.shape
    rows, cols = binary.any(-1), binary.any(-2)
    ys, xs = torch.arange(H), torch.arange(W)
    top = torch.where(rows, ys, H).min(-1).values
    bottom = torch.where(rows, ys, -1).max(-1).values
    left = torch.where(cols, xs, W).min(-1).values
    right = torch.where(cols, xs, -1).max(-1).values
    boxes = torch.stack([left, top, right, bottom], dim=-1)
    boxes = torch.where((mid > 0)[:, None], boxes, torch.zeros_like(boxes))
    return dict(count_hi=hi, count_lo=lo, count=mid, stability=hi / lo, boxes=boxes.long(), binary=binary)


def nms(boxes: torch.Tensor, scores: torch.Tensor, iou_threshold: float) -> torch.Tensor:
    """torchvision batched_nms with one class (P:715-720): greedy in descending score order (ties by index), a box
    suppresses later ones whose IoU (fp32, areas without +1) exceeds the threshold.  -> kept indices, keep order."""
    boxes = boxes.float()
    order = torch.sort(scores, descending=True, stable=True).indices
    b = boxes[order]
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    removed = torch.zeros(len(order), dtype=torch.bool)
    keep = []
    for i in range(len(order)):
        if removed[i]:
            continue
        keep.append(int(order[i]))
        w = (torch.minimum(b[i, 2], b[i + 1:, 2]) - torch.maximum(b[i, 0], b[i + 1:, 0])).clamp(min=0)
        h = (torch.minimum(b[i, 3], b[i + 1:, 3]) - torch.maximum(b[i, 1], b[i + 1:, 1])).clamp(min=0)
        inter = w * h
        iou = inter / (area[i] + area[i + 1:] - inter)
        removed[i + 1:] |= iou.double() > iou_threshold
    return torch.tensor(keep, dtype=torch.int64)


def generate(low_res: torch.Tensor, iou_scores: torch.Tensor, original_size: tuple, reshaped_size: tuple,
             pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0,
             mask_threshold: float = 0.0, crops_nms_thresh: float = 0.7, pad_size=(1024, 1024)) -> dict:
    """Steps 3-6 of the pipeline for one image (G:277-294 and G:312-321): low_res fp32 [n_points, 3, hm, wm] and
    iou_scores [n_points, 3] of every point prompt -> candidates flattened point-major (filter_masks' flatten(0, 1),
    P:337-338), filtered by each enabled threshold (P:350-356), boxed (P:362-363), de-duplicated.
    -> dict(index = kept candidate indices in keep order, scores, stability, boxes int64, masks bool [k, H, W], and
    the candidate count after each stage: candidates, after_iou, after_stability, after_nms)."""
    masks = upscale(low_res, original_size, reshaped_size, pad_size).flatten(0, 1)
    iou = iou_scores.flatten(0, 1).float()
    st = mask_stats(masks, mask_threshold, stability_score_offset)
    keep = torch.ones(len(iou), dtype=torch.bool)
    if pred_iou_thresh > 0.0:
        keep &= iou > pred_iou_thresh
    after_iou = int(keep.sum())
    if stability_score_thresh > 0.0:
        keep &= st["stability"] > stability_score_thresh
    cand = torch.nonzero(keep).view(-1)
    kept = nms(st["boxes"][cand], iou[cand], crops_nms_thresh)
    index = cand[kept]
    return dict(index=index, scores=iou[index], stability=st["stability"][index], boxes=st["boxes"][index],
                masks=st["binary"][index], candidates=len(iou), after_iou=after_iou, after_stability=len(cand),
                after_nms=len(index), stats=st)
