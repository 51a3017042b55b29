"""Plain-torch restatement of the query detectors' panoptic output: MaskFormerFusionHead.panoptic_postprocess
(mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py:41-106) and RSMaskFormerFusionHead.predict
(M:663-715) with its panoptic branch.  The arithmetic is the reference's (fp32 sigmoid, product with the score, argmax
over the kept queries, Python division of the two counts); it runs on CPU or CUDA tensors alike."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .restate_query import fusion_rescale, instance_postprocess

INSTANCE_OFFSET = 1000      # mmdet/evaluation/functional/panoptic_utils.py


def panoptic_postprocess(mask_cls: torch.Tensor, mask_pred: torch.Tensor, num_classes: int, num_things_classes: int,
                         test_cfg: dict, stats: bool = False):
    """maskformer_fusion_head.py:41-106, one image: mask_cls [nq, C+1], mask_pred [nq, h, w] logits at the output size
    -> int32 [1, h, w]; with ``stats`` also dict(query, mask_area, original_area, segment_id) of the kept queries in
    kept order (segment_id -1 for a skipped query)."""
    object_mask_thr = test_cfg.get("object_mask_thr", 0.8)          # :58-60
    iou_thr = test_cfg.get("iou_thr", 0.8)
    filter_low_score = test_cfg.get("filter_low_score", False)
    scores, labels = F.softmax(mask_cls, dim=-1).max(-1)            # :62
    masks = mask_pred.sigmoid()                                     # :63
    keep = labels.ne(num_classes) & (scores > object_mask_thr)      # :65
    cur_scores, cur_classes, cur_masks = scores[keep], labels[keep], masks[keep]
    cur_prob_masks = cur_scores.view(-1, 1, 1) * cur_masks          # :70
    h, w = cur_masks.shape[-2:]
    pan = torch.full((h, w), num_classes, dtype=torch.int32, device=cur_masks.device)
    st = dict(query=torch.nonzero(keep).flatten().tolist(), mask_area=[], original_area=[], segment_id=[])
    if cur_masks.shape[0]:
        ids = cur_prob_masks.argmax(0)                              # :81, the first kept query on ties
        instance_id = 1
        for k in range(cur_classes.shape[0]):                       # :83-104
            pred_class = int(cur_classes[k].item())
            mask = ids == k
            mask_area = mask.sum().item()
            original_area = (cur_masks[k] >= 0.5).sum().item()
            if filter_low_score:
                mask = mask & (cur_masks[k] >= 0.5)
            seg = -1
            if mask_area > 0 and original_area > 0 and not mask_area / original_area < iou_thr:
                if pred_class >= num_things_classes:                # stuff: one id per class, regions merge
                    seg = pred_class
                else:
                    seg = pred_class + instance_id * INSTANCE_OFFSET
                    instance_id += 1
                pan[mask] = seg
            st["mask_area"].append(int(mask_area))
            st["original_area"].append(int(original_area))
            st["segment_id"].append(seg)
    return (pan[None], st) if stats else pan[None]


def fusion_predict(mask_cls: torch.Tensor, mask_pred: torch.Tensor, metas: list, num_classes: int,
                   num_things_classes: int, test_cfg: dict, rescale: bool = False) -> list:
    """RSMaskFormerFusionHead.predict (M:663-715): mask_cls [B, nq, C+1], mask_pred [B, nq, Hb, Wb] (after the
    M:652-656 up-sampling); per image crop to int(ori * scale_factor), with ``rescale`` bilinear to ori_shape, then the
    panoptic (default on) and instance (default off) branches.  Semantic output is refused, as in the reference."""
    assert not test_cfg.get("semantic_on", False), "semantic segmentation results are not supported"
    out = []
    for cls, mp, meta in zip(mask_cls, mask_pred, metas):
        ori_h, ori_w = meta["ori_shape"][:2]
        sf = meta["scale_factor"]
        mp = mp[:, :int(ori_h * sf[1]), :int(ori_w * sf[0])]       # :681-686
        if rescale:                                                 # :688-695
            mp = F.interpolate(mp[:, None], size=(ori_h, ori_w), mode="bilinear", align_corners=False)[:, 0]
        r = {}
        if test_cfg.get("panoptic_on", True):
            r["pan_results"] = panoptic_postprocess(cls, mp, num_classes, num_things_classes, test_cfg)
        if test_cfg.get("instance_on", False):
            r["ins_results"] = instance_postprocess(cls, mp, num_classes, test_cfg.get("max_per_image", 100))
        out.append(r)
    return out


def resample(logits: torch.Tensor, size: tuple, meta: dict | None = None, rescale: bool = True) -> torch.Tensor:
    """The masks the panoptic step sees, from the head's low-res logits [nq, hm, wm]: bilinear to the batch shape
    ``size`` (M:652-656), and for a resized / padded image the crop and, with ``rescale``, the resize to ori_shape
    (M:679-691)."""
    if meta is None:
        return F.interpolate(logits[None], size=tuple(size), mode="bilinear", align_corners=False)[0]
    return fusion_rescale(logits, dict(meta, batch_input_shape=tuple(size)), rescale=rescale)
