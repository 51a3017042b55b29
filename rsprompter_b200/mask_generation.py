"""Segment everything with SAM on the GPU: HF transformers' ``pipeline("mask-generation")`` for one crop layer.

HF's MaskGenerationPipeline (pipelines/mask_generation.py:187-335) prompts the model with a regular point grid, turns
every candidate mask into an fp32 mask at the original image size (SamImageProcessor.post_process_masks(binarize=False),
image_processing_sam.py:379-430), filters it by predicted IoU and stability score, boxes it (filter_masks :301-377) and
de-duplicates with a box NMS (post_process_for_mask_generation :432-446).  Here:

  * every image of the call is encoded in one batch, and the grids of all images run through the mask decoder in
    calls of ``points_per_batch`` prompts (prompts of several images share a call through the decoder's block maps);
  * ``rsp_sam_mask_stats`` reduces each call's low-res logits to three pixel counts, a box and the keep flag,
    sampling every original-size pixel with the two-resizes-and-crop sampler of ``rsp_mask_paste``:
    the original-size fp32 mask never exists;
  * one ``rsp_nms_batched`` + ``rsp_compact_keep`` per call de-duplicates every image's survivors, ties broken by
    candidate order (point-major, mask-minor, HF's ``flatten(0, 1)``);
  * only the kept masks are pasted, as bits, by ``rsp_mask_paste``; ``output_rle_mask=True`` encodes
    them as COCO RLE on the GPU.

The low-res logits of every candidate of every image of the call stay on the device until the NMS has run: 256 KB
per candidate, 3 per point, 805 MB per image at the default 32 x 32 grid, so a call on B images holds B times that at
once (pass fewer images per call to bound it).  Host synchronisations per call: the read of the kept counts and
candidates, two more with ``output_rle_mask`` and one more with ``min_mask_region_area`` > 0 (none when no mask is
kept), whatever the grid size and the number of masks.

``crops_n_layers > 0`` is not built: HF's own crop path cannot run (``_generate_crop_boxes`` stacks crops of different
sizes), so there are no reference semantics for it.  HF's ``max_hole_area`` / ``max_sprinkle_area`` are not built
either (HF's SAM processor has no such arguments and its SAM2 processor ignores them).  SAM's ``min_mask_region_area``
is: ``rsp_mask_small_regions_bits`` fills small holes and removes small islands of the kept masks on the GPU (connected
components of the bit-packed masks by a block-based union-find), and a second ``rsp_nms_batched`` ranks the masks it
changed after those it left alone: one more host synchronisation per call.

``generate_scene_masks`` runs the same stages over the overlapping windows of a whole scene (large_image's slicing),
with HF's crop-edge rule applied in ``rsp_sam_mask_stats``, RLE of the whole scene from each window's bits, and
one cross-window box NMS; ``coarse_patch_sizes`` adds layers of larger windows up to the whole scene, resized by
``rsp_resize_aa_pad_u8`` (SamImageProcessor's antialiased resize) and merged under the finer layers as SAM merges
its crop layers.

``python -m rsprompter_b200.mask_generation IMAGE --arch base --checkpoint sam.safetensors --out masks.json`` writes
one dict per mask (COCO RLE ``segmentation``, xywh ``bbox``, ``predicted_iou``, ``stability_score``,
``point_coords``); with ``--patch-size P`` the image is a scene cut into P x P windows, and each dict also has the
window's ``crop_box``; ``--coarse-patch-sizes P1 [P2 ...]`` adds layers of coarser windows up to the whole scene,
and each dict then has its ``layer``."""
from __future__ import annotations

import argparse
import json
import math
import numbers

import torch

from . import _lib
from .geojson import feature_collection

# SamImageProcessor defaults (image_processing_sam.py:61-75): ImageNet mean / std on [0, 1] pixels
IMAGE_MEAN = (0.485, 0.456, 0.406)
IMAGE_STD = (0.229, 0.224, 0.225)

CROP_ERROR = ("crops_n_layers > 0 is not supported: HF's own crop path cannot run (_generate_crop_boxes torch.stack()s "
              "crops of different sizes and fails with 'stack expects each tensor to be equal size'), so there are no "
              "reference semantics to follow")


def preprocess_shape(hw: tuple, longest_edge: int) -> tuple:
    """SamImageProcessor._get_preprocess_shape (image_processing_sam.py:113-122): the resized, unpadded (h, w)."""
    oldh, oldw = int(hw[0]), int(hw[1])
    scale = longest_edge * 1.0 / max(oldh, oldw)
    return int(oldh * scale + 0.5), int(oldw * scale + 0.5)


def point_grid(points_per_side: int, hw: tuple, target_size: int) -> tuple:
    """The prompts of one image: _build_point_grid (image_processing_sam.py:624-631) scaled by (W, H) as
    _generate_crop_images does for the whole-image crop (:649-653), then _normalize_coordinates (:659-684) into the
    model frame.  -> (points in original pixels, points in the model frame), fp32 [n * n, 2] on the host."""
    offset = 1 / (2 * points_per_side)
    side = torch.linspace(offset, 1 - offset, points_per_side)
    grid = torch.stack([torch.tile(side[None, :], (points_per_side, 1)), torch.tile(side[:, None], (1, points_per_side))],
                       dim=-1).reshape(-1, 2)
    H, W = int(hw[0]), int(hw[1])
    pts = grid * torch.tensor([H, W]).flip(dims=(0,)).unsqueeze(0)
    new_h, new_w = preprocess_shape((H, W), target_size)
    model = pts.clone().float()
    model[..., 0] = model[..., 0] * (new_w / W)
    model[..., 1] = model[..., 1] * (new_h / H)
    return pts, model


def _check_params(points_per_side, points_per_batch, crops_n_layers, max_hole_area, max_sprinkle_area) -> None:
    if crops_n_layers:
        raise ValueError(CROP_ERROR)
    if max_hole_area is not None or max_sprinkle_area is not None:
        raise ValueError("max_hole_area / max_sprinkle_area are not supported: SamImageProcessor.post_process_masks "
                         "takes no hole or sprinkle arguments")
    if points_per_batch is None or points_per_batch <= 0:
        raise ValueError("Cannot have points_per_batch<=0. Must be >=1 to returned batched outputs.")
    if points_per_side is None or points_per_side < 1:
        raise ValueError(f"points_per_side must be >= 1, got {points_per_side}")


def _sam(model):
    from .sam_model import RSSamModel, SamModelB200
    if isinstance(model, RSSamModel):
        return model.sam_model
    if isinstance(model, SamModelB200):
        return model
    raise TypeError(f"generate_masks takes an RSSamModel or SamModelB200, not {type(model).__name__}")


def _sizes(v, B: int, name: str) -> list:
    if v is None:
        raise ValueError(f"pixel_values needs {name}: one (h, w) per image, as SamProcessor returns them")
    v = v.tolist() if isinstance(v, torch.Tensor) else list(v)
    if len(v) != B:
        raise ValueError(f"{name} has {len(v)} entries for {B} images")
    return [(int(h), int(w)) for h, w in v]


def _inputs(sam, images, pixel_values, original_sizes, reshaped_input_sizes, dev, antialias: bool = False):
    """-> (pixel_values fp32 [B, 3, S, S] on dev, original (h, w) per image, reshaped (h, w) per image).  Images are
    resized by rsp_resize_pad_u8, or with ``antialias`` by rsp_resize_aa_pad_u8 (SamImageProcessor's resize)."""
    S = sam.varch.image_size
    if (images is None) == (pixel_values is None):
        raise ValueError("pass exactly one of images and pixel_values")
    if pixel_values is not None:
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, S, S):
            raise ValueError(f"pixel_values must be [B, 3, {S}, {S}], got {tuple(pixel_values.shape)}")
        B = pixel_values.shape[0]
        sizes = _sizes(original_sizes, B, "original_sizes")
        reshaped = _sizes(reshaped_input_sizes, B, "reshaped_input_sizes")
        for rs in reshaped:
            if not (0 < rs[0] <= S and 0 < rs[1] <= S):
                raise ValueError(f"reshaped input size {rs} is outside the {S} x {S} input")
        return pixel_values.to(dev, torch.float32).contiguous(), sizes, reshaped
    imgs = [images] if isinstance(images, torch.Tensor) and images.dim() == 3 else list(images)
    if not imgs:
        raise ValueError("no images")
    for t in imgs:
        if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[0] != 3:
            raise ValueError("images must be uint8 RGB tensors [3, H, W]")
    sizes = [(int(t.shape[1]), int(t.shape[2])) for t in imgs]
    reshaped = [preprocess_shape(hw, S) for hw in sizes]
    views = [t if t.device == dev else t.contiguous().pin_memory().to(dev, non_blocking=True) for t in imgs]
    mean = tuple(255.0 * m for m in IMAGE_MEAN)
    std = tuple(255.0 * s for s in IMAGE_STD)
    pix = torch.empty(len(imgs), 3, S, S, device=dev, dtype=torch.float32)
    resize = _lib.resize_aa_pad_u8 if antialias else _lib.resize_pad_u8
    resize(views, reshaped, pix, mean, std, False, mean)                  # padded with the mean: 0 once normalised
    return pix, sizes, reshaped


def _candidates(sam, emb_nhwc, sizes, reshaped, p, crops=None) -> dict:
    """The grids of every image through the decoder in calls of points_per_batch prompts, each call's logits through
    rsp_sam_mask_stats.  -> per-candidate device tensors, candidate c of image b at [b, c] (point c // 3, mask c % 3).
    ``crops``: per image, ((x0, y0, x1, y1), (H, W)) when it is that crop box of an H x W scene; the keep flags then
    include the crop-edge rule (rsp_sam_mask_stats with scene_h > 0)."""
    B, g, C = emb_nhwc.shape[0], emb_nhwc.shape[1], emb_nhwc.shape[3]
    S = sam.varch.image_size
    dev = emb_nhwc.device
    n_pts = p["points_per_side"] ** 2
    grids = [point_grid(p["points_per_side"], hw, S) for hw in sizes]
    pts_orig = torch.stack([a for a, _ in grids]).pin_memory().to(dev, non_blocking=True)       # [B, n_pts, 2]
    pts_model = torch.stack([b for _, b in grids]).view(1, B * n_pts, 1, 2).pin_memory().to(dev, non_blocking=True)
    labels = torch.ones(1, B * n_pts, 1, dtype=torch.int32, device=dev)
    sparse = sam.embed_points(pts_model, labels, pad=True).reshape(B * n_pts, 2, C).contiguous()
    prompt_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(n_pts)
    pos_rows = sam.shared_image_embedding.image_wide_rows(g)
    dense = sam.prompt_encoder.no_mask_embed.weight[0].to(torch.float32).contiguous()
    emb_rows = emb_nhwc.reshape(B, g * g, C)
    hm = wm = 4 * g
    n_out = sam.mask_decoder.num_mask_tokens - 1
    Nc = n_pts * n_out
    logits = torch.empty(B * Nc, hm, wm, device=dev, dtype=torch.float32)
    iou = torch.empty(B * Nc, device=dev, dtype=torch.float32)
    stab = torch.empty(B * Nc, device=dev, dtype=torch.float32)
    boxes = torch.empty(B * Nc, 4, device=dev, dtype=torch.int32)
    keep = torch.empty(B * Nc, device=dev, dtype=torch.bool)
    ppb = p["points_per_batch"]
    for q0 in range(0, B * n_pts, ppb):
        q1 = min(q0 + ppb, B * n_pts)
        b0, b1 = q0 // n_pts, (q1 - 1) // n_pts + 1             # the images this call's prompts belong to
        m, s = sam.mask_decoder.decode(emb_rows[b0:b1].reshape(-1, C), pos_rows, sparse[q0:q1], (g, g),
                                       prompt_img=(prompt_img[q0:q1] - b0).contiguous(), dense_vec=dense,
                                       multimask_output=True)
        logits[q0 * n_out:q1 * n_out].copy_(m.view(-1, hm, wm))
        iou[q0 * n_out:q1 * n_out].copy_(s.reshape(-1))
        for b in range(b0, b1):
            r0, r1 = max(q0, b * n_pts) * n_out, min(q1, (b + 1) * n_pts) * n_out
            _, bx, st, kp = _lib.sam_mask_stats(
                logits[r0:r1], ((S, S), reshaped[b], sizes[b]), p["mask_threshold"], p["stability_score_offset"],
                iou[r0:r1], p["pred_iou_thresh"], p["stability_score_thresh"], crop=None if crops is None else crops[b])
            boxes[r0:r1].copy_(bx)
            stab[r0:r1].copy_(st)
            keep[r0:r1].copy_(kp)
    return dict(logits=logits, iou=iou.view(B, Nc), stability=stab.view(B, Nc), boxes=boxes.view(B, Nc, 4),
                keep=keep.view(B, Nc), points=pts_orig, n_out=n_out, sizes=sizes, reshaped=reshaped)


def _nms(iou: torch.Tensor, keep: torch.Tensor, boxes: torch.Tensor, iou_thr: float) -> tuple:
    """batched_nms(boxes.float(), scores, zeros, iou_thr) over every image's survivors (post_process_for_mask_generation,
    image_processing_sam.py:715-720), in keep order: scores iou fp32 [B, Nc], survivors keep bool [B, Nc], boxes
    [B, Nc, 4].  -> (kept index int64 [B, Nc] on the device, kept count per image on the host, the same indices on the
    host); one host synchronisation."""
    B, Nc = iou.shape
    key = torch.where(keep, iou, torch.full_like(iou, -float("inf")))
    _, order = torch.sort(key, dim=1, descending=True, stable=True)     # survivors first; ties by candidate order
    nvalid = keep.sum(1).to(torch.int32)
    boxes_s = torch.gather(boxes.float(), 1, order[..., None].expand(-1, -1, 4)).contiguous()
    scores_s = torch.gather(iou, 1, order).contiguous()
    ids = torch.zeros(B, Nc, device=iou.device, dtype=torch.int64)
    kept = _lib.nms_batched(boxes_s, ids, nvalid, iou_thr)
    _, _, _, oi, cnt = _lib.compact_keep(kept, boxes_s, scores_s, None, Nc)
    idx = torch.gather(order, 1, oi.clamp(min=0).long())
    host = torch.cat([cnt.long(), idx.view(-1)]).cpu()
    return idx, host[:B].tolist(), host[B:].view(B, Nc)


def _paste(cand: dict, b: int, ci: torch.Tensor, mask_threshold: float, target_size: int) -> torch.Tensor:
    """The candidates ci (device indices) of image b pasted as bits at the image's original size."""
    Nc = cand["iou"].shape[1]
    H, W = cand["sizes"][b]
    bits = torch.empty(ci.shape[0], H, (W + 15) // 16 * 2, device=ci.device, dtype=torch.uint8)
    if ci.shape[0]:
        lg = cand["logits"].index_select(0, ci + b * Nc)
        _lib.mask_paste(lg, mask_threshold, raw=True, rescale=((target_size, target_size), cand["reshaped"][b], (H, W)),
                        bits=bits)
    return bits


def _outputs(cand: dict, idx: torch.Tensor, counts: list, idx_host: torch.Tensor, mask_threshold: float,
             target_size: int) -> list:
    """Per image: the kept masks pasted as bits, and the kept rows of every per-candidate output."""
    B, Nc = cand["iou"].shape
    out = []
    for b in range(B):
        k = counts[b]
        H, W = cand["sizes"][b]
        ci = idx[b, :k]
        bits = _paste(cand, b, ci, mask_threshold, target_size)
        out.append(dict(masks=bits, scores=cand["iou"][b].index_select(0, ci),
                        stability_scores=cand["stability"][b].index_select(0, ci),
                        boxes=cand["boxes"][b].index_select(0, ci).long(),
                        points=cand["points"][b].index_select(0, ci // cand["n_out"]),
                        candidates=idx_host[b, :k].clone(), size=(H, W)))
    return out


# Device bytes of the label workspace of one rsp_mask_small_regions_bits launch (4 bytes per 2 x 2 pixel block, 1 MB
# per 1024 x 1024 mask): masks are cleaned in chunks that fit, with results independent of the chunk size.
SMALL_REGIONS_WORKSPACE_BYTES = 256 << 20


def _check_region_area(min_mask_region_area) -> float:
    a = float(min_mask_region_area)
    if not math.isfinite(a):
        raise ValueError(f"min_mask_region_area must be finite, got {min_mask_region_area}")
    return a


def _clean(bits: torch.Tensor, W: int, min_area: float) -> tuple:
    """rsp_mask_small_regions_bits' holes then islands on the masks bits uint8 [k, H, ld] (k > 0), in place, in chunks
    whose label workspace fits SMALL_REGIONS_WORKSPACE_BYTES.  -> (unchanged fp32 [k], 1 for a mask neither step
    changed, boxes int32 [k, 4] of the cleaned masks)."""
    k, H = bits.shape[0], bits.shape[1]
    # areas are integers, so "< A" is "< ceil(A)"; every A above H * W (one more than the largest area) gives the
    # same result, and the clamp keeps a huge finite A within the kernel's 64-bit threshold
    thr = min(math.ceil(min_area), H * W + 1)
    chunk = max(1, SMALL_REGIONS_WORKSPACE_BYTES // _lib.small_regions_ws_bytes(1, H, W))
    ws = torch.empty(_lib.small_regions_ws_bytes(min(chunk, k), H, W), device=bits.device, dtype=torch.uint8)
    tmp = torch.empty_like(bits[:chunk])
    unchanged = torch.empty(k, device=bits.device, dtype=torch.float32)
    boxes = torch.empty(k, 4, device=bits.device, dtype=torch.int32)
    for j0 in range(0, k, chunk):
        j1 = min(j0 + chunk, k)
        part = bits[j0:j1]
        _, ch_h, _ = _lib.mask_small_regions_bits(part, W, thr, "holes", out=tmp[:j1 - j0], ws=ws)
        _, ch_i, bx = _lib.mask_small_regions_bits(tmp[:j1 - j0], W, thr, "islands", out=part, ws=ws)
        unchanged[j0:j1] = (~(ch_h | ch_i)).float()
        boxes[j0:j1] = bx
    return unchanged, boxes


def _remove_small_regions(out: list, min_area: float, iou_thr: float) -> list:
    """SAM's postprocess_small_regions (min_mask_region_area) on every image's kept masks: holes then islands by
    rsp_mask_small_regions_bits, the boxes of the cleaned masks, and a box NMS with score float(unchanged) at iou_thr
    through _nms.  Ties keep the first NMS's order (a stable sort; SAM's torchvision sort is not stable).  -> the
    results in the new keep order, ``masks`` and ``boxes`` those of the cleaned masks; one host synchronisation."""
    K = max(r["masks"].shape[0] for r in out)
    if K == 0:
        return out
    dev = out[0]["masks"].device
    B = len(out)
    unchanged = torch.zeros(B, K, device=dev, dtype=torch.float32)
    valid = torch.zeros(B, K, device=dev, dtype=torch.bool)
    boxes = torch.zeros(B, K, 4, device=dev, dtype=torch.int32)
    for b, r in enumerate(out):
        k = r["masks"].shape[0]
        if k == 0:
            continue
        unchanged[b, :k], boxes[b, :k] = _clean(r["masks"], r["size"][1], min_area)
        valid[b, :k] = True
    idx, counts, idx_host = _nms(unchanged, valid, boxes, iou_thr)
    res = []
    for b, r in enumerate(out):
        rows = idx[b, :counts[b]]
        res.append(dict(masks=r["masks"].index_select(0, rows), scores=r["scores"].index_select(0, rows),
                        stability_scores=r["stability_scores"].index_select(0, rows),
                        boxes=boxes[b].index_select(0, rows).long(), points=r["points"].index_select(0, rows),
                        candidates=r["candidates"][idx_host[b, :counts[b]]], size=r["size"]))
    return res


def _add_rle(out: list, places: list | None = None, rle: bool = True, polygons: bool = False) -> None:
    """COCO RLE strings (``rle``) and polygons (``polygons``) of every image's masks, each in one batch on the GPU from
    the same placed descriptors.  ``places``: per image, (SH, SW, y0, x0) to encode its masks as masks of an SH x SW
    canvas that is zero but for the image at (y0, x0).  Polygons are (contours, hierarchy) of cv2.findContours(canvas,
    RETR_CCOMP, CHAIN_APPROX_SIMPLE): int32 [k, 2] (x, y) canvas pixel indices and int32 [1, n, 4] (None when empty)."""
    rle_groups, sizes = [], []
    for b, r in enumerate(out):
        bits = r["masks"]
        k, (H, W) = bits.shape[0], r["size"]
        SH, SW, y0, x0 = (H, W, 0, 0) if places is None else places[b]
        sizes.append([SH, SW])
        if k:
            ld = bits.shape[2]
            rle_groups.append((bits, [(j * H * ld, ld, H, H, W, SH, SW, y0, x0) for j in range(k)]))
    if rle:
        strings = iter(_lib.mask_rle_placed(rle_groups, packed=True))
        for r, size in zip(out, sizes):
            r["rle"] = [dict(size=list(size), counts=next(strings)) for _ in range(r["masks"].shape[0])]
    if polygons:
        canvases = [(SH, SW, [(g, off, ld, rows, h, w, y0, x0)])
                    for g, (_, pl) in enumerate(rle_groups) for off, ld, rows, h, w, SH, SW, y0, x0 in pl]
        polys = iter(_lib.mask_contours([bits for bits, _ in rle_groups], canvases, _lib.CHAIN_APPROX_SIMPLE))
        for r in out:
            r["polygons"] = [next(polys) for _ in range(r["masks"].shape[0])]


@torch.no_grad()
def generate_masks(model, images=None, *, pixel_values=None, original_sizes=None, reshaped_input_sizes=None,
                   points_per_side: int = 32, points_per_batch: int = 64, pred_iou_thresh: float = 0.88,
                   stability_score_thresh: float = 0.95, stability_score_offset: float = 1.0,
                   mask_threshold: float = 0.0, crops_nms_thresh: float = 0.7, crops_n_layers: int = 0,
                   max_hole_area=None, max_sprinkle_area=None, min_mask_region_area: float = 0,
                   output_rle_mask: bool = False, output_polygons: bool = False) -> list:
    """Every mask of each image, as HF's mask-generation pipeline finds them with crops_n_layers=0.

    ``model``: an RSSamModel or SamModelB200.  Images go in one of two forms:

      * ``images``: uint8 RGB [3, H, W] tensors (one, or a list of any sizes, on the host or the device), resized by
        ``rsp_resize_pad_u8`` to SamImageProcessor's size (longest edge = the model's image size), normalised with its
        ImageNet mean and std (x 255) and padded with 0 to the square input.  The resize is cv2 ``INTER_LINEAR``
        arithmetic (this project's and mmdet's), not the antialiased bilinear resize of torchvision that
        SamImageProcessor runs, so the pixel values are close to HF's but not the same bytes;
      * ``pixel_values`` fp32 [B, 3, S, S] with ``original_sizes`` and ``reshaped_input_sizes`` (one (h, w) per
        image): exactly what SamProcessor returns, for results comparable to HF's.

    Parameters carry HF's names and defaults (``points_per_side`` is HF's ``points_per_crop``); a threshold of 0
    disables its test, as in filter_masks.  ``crops_n_layers > 0``, ``max_hole_area`` and ``max_sprinkle_area`` raise
    ValueError.

    ``min_mask_region_area`` = A > 0 is SAM's (SamAutomaticMaskGenerator.postprocess_small_regions) on the kept masks
    at their original size: 8-connected background components of area < A are filled (border ones included), then of
    the foreground components only those of area >= A are kept, or the largest alone when none is (ties: cv2's label
    order).  Masks are then boxed again and go through a second box NMS at ``crops_nms_thresh`` with score 1 for a
    mask that neither step changed and 0 otherwise, so unchanged masks come first.  A step counts as a change when it
    finds a small component, as in SAM, even if the mask stays the same.  Ties keep the first NMS's order: this sort is
    stable, SAM's torchvision sort is not.  A <= 0 (SAM's default) skips the step; a non-finite A raises ValueError.

    Returns one dict per image, rows in NMS keep order (descending predicted IoU; with min_mask_region_area, the
    order of the second NMS):
      masks             uint8 [k, H, ceil(W / 16) * 2] bit-packed rows, pixel x = bit x % 8 of byte x // 8
                        (``masks_to_bool`` unpacks them)
      scores            fp32 [k] predicted IoU
      stability_scores  fp32 [k]
      boxes             int64 [k, 4] inclusive pixel xyxy (HF's _batched_mask_to_box)
      points            fp32 [k, 2] the prompt of each mask, in original pixels
      candidates        int64 [k] (host) candidate index: point * 3 + output mask
      size              (H, W)
      rle               with output_rle_mask: COCO compressed RLE dicts {'size': [H, W], 'counts': bytes}
      polygons          with output_polygons: per mask (contours, hierarchy), cv2.findContours(mask, RETR_CCOMP,
                        CHAIN_APPROX_SIMPLE) traced on the GPU from the same bits (two host synchronisations)
    All tensors but ``candidates`` are on the model's device.

    Memory: the low-res logits of every candidate of every image stay resident until the NMS, 3 x points_per_side^2 x
    256 KB per image (805 MB at the default grid), so B images in one call need B times that at once."""
    _check_params(points_per_side, points_per_batch, crops_n_layers, max_hole_area, max_sprinkle_area)
    min_area = _check_region_area(min_mask_region_area)
    sam = _sam(model)
    dev = sam.prompt_encoder.no_mask_embed.weight.device
    pix, sizes, reshaped = _inputs(sam, images, pixel_values, original_sizes, reshaped_input_sizes, dev)
    p = dict(points_per_side=int(points_per_side), points_per_batch=int(points_per_batch),
             pred_iou_thresh=float(pred_iou_thresh), stability_score_thresh=float(stability_score_thresh),
             stability_score_offset=float(stability_score_offset), mask_threshold=float(mask_threshold))
    emb = sam._encode(pix)
    cand = _candidates(sam, emb, sizes, reshaped, p)
    idx, counts, idx_host = _nms(cand["iou"], cand["keep"], cand["boxes"], float(crops_nms_thresh))
    out = _outputs(cand, idx, counts, idx_host, float(mask_threshold), sam.varch.image_size)
    if min_area > 0:
        out = _remove_small_regions(out, min_area, float(crops_nms_thresh))
    if output_rle_mask or output_polygons:
        _add_rle(out, rle=output_rle_mask, polygons=output_polygons)
    return out


def scene_crop_boxes(hw: tuple, patch_size: int, overlap_ratio: float) -> list:
    """The windows of generate_scene_masks over an H x W scene: large_image.slice_origins' P x P windows, each cut to
    its in-scene part, as crop boxes (x0, y0, min(x0 + P, W), min(y0 + P, H)) in slice order."""
    from .large_image import slice_origins
    H, W = int(hw[0]), int(hw[1])
    P = int(patch_size)
    return [(x0, y0, min(x0 + P, W), min(y0 + P, H)) for x0, y0 in slice_origins((H, W), P, overlap_ratio)]


def scene_layer_windows(hw: tuple, patch_size: int, overlap_ratio: float, coarse_patch_sizes=()) -> list:
    """The windows of every layer of generate_scene_masks: [(layer, crop boxes)], layer 0 the base windows of
    ``patch_size``, layer l those of coarse_patch_sizes[l - 1] (scene_crop_boxes of each size; a size >= max(H, W)
    is one window, the scene).  A layer whose windows are those of the previous layer that runs is left out."""
    out = [(0, scene_crop_boxes(hw, patch_size, overlap_ratio))]
    for l, p in enumerate(coarse_patch_sizes, 1):
        boxes = scene_crop_boxes(hw, p, overlap_ratio)
        if boxes != out[-1][1]:
            out.append((l, boxes))
    return out


def _coarse_sizes(coarse_patch_sizes, hw: tuple) -> list:
    sizes = []
    for v in coarse_patch_sizes:
        if isinstance(v, bool) or not isinstance(v, numbers.Integral):
            raise ValueError(f"coarse_patch_sizes must be integers, got {v!r}")
        sizes.append(int(v))
    if any(b <= a for a, b in zip(sizes, sizes[1:])):
        raise ValueError(f"coarse_patch_sizes must be strictly increasing, got {tuple(sizes)}")
    H, W = hw
    for c in sizes:
        if min(c, H) * min(c, W) >= 1 << 31:
            raise ValueError(f"a {min(c, H)} x {min(c, W)} window of coarse patch size {c} has 2^31 pixels or more, "
                             f"beyond the mask statistics and RLE kernels")
    return sizes


# Device bytes of the bit-packed masks one batch of coarse-layer windows holds at once.  A coarse window's masks are
# large (P^2 / 8 bytes each, H * W / 8 for the whole scene: 50 MB at 20 000^2), so they are pasted, cleaned and
# encoded in chunks of at most this many bytes (at least one mask), with results independent of the chunk size.
COARSE_MASK_BYTES = 1 << 30


def _chunks(counts: list, per_mask: list, budget: int) -> list:
    """Every window's kept rows as consecutive (window, j0, j1) segments, grouped so that one group's masks take at most
    ``budget`` bytes (at least one mask per group)."""
    groups, cur, used = [], [], 0
    for b, k in enumerate(counts):
        j = 0
        while j < k:
            room = (budget - used) // per_mask[b]
            if room == 0 and cur:
                groups.append(cur)
                cur, used = [], 0
                continue
            j1 = min(k, j + max(room, 1))
            cur.append((b, j, j1))
            used += (j1 - j) * per_mask[b]
            j = j1
    if cur:
        groups.append(cur)
    return groups


def _coarse_outputs(cand: dict, idx: torch.Tensor, counts: list, idx_host: torch.Tensor, p: dict, target_size: int,
                    min_area: float, nms_thr: float, places: list, polygons: bool = False) -> list:
    """_outputs, then _remove_small_regions with min_area > 0, then _add_rle(places), for a batch of coarse-layer
    windows, with the kept masks pasted, cleaned and encoded in groups of at most COARSE_MASK_BYTES: the same rows and
    strings, without the masks.  Host synchronisations: the RLE's per group, one more for the second NMS."""
    B = len(counts)
    dev = idx.device
    per_mask = [H * ((W + 15) // 16 * 2) for H, W in cand["sizes"]]
    K = max(counts)
    unchanged = torch.zeros(B, K, device=dev, dtype=torch.float32)
    valid = torch.zeros(B, K, device=dev, dtype=torch.bool)
    boxes = cand["boxes"].gather(1, idx[:, :K, None].expand(-1, -1, 4)).contiguous()
    rle = [[] for _ in range(B)]
    polys = [[] for _ in range(B)]
    for group in _chunks(counts, per_mask, COARSE_MASK_BYTES):
        parts = []
        for b, j0, j1 in group:
            bits = _paste(cand, b, idx[b, j0:j1], p["mask_threshold"], target_size)
            if min_area > 0:
                unchanged[b, j0:j1], boxes[b, j0:j1] = _clean(bits, cand["sizes"][b][1], min_area)
            parts.append(dict(masks=bits, size=cand["sizes"][b]))
        _add_rle(parts, places=[places[b] for b, _, _ in group], polygons=polygons)
        for (b, _, _), r in zip(group, parts):
            rle[b].extend(r["rle"])
            polys[b].extend(r.get("polygons", ()))
    out = []
    for b in range(B):
        k = counts[b]
        ci = idx[b, :k]
        valid[b, :k] = True
        out.append(dict(scores=cand["iou"][b].index_select(0, ci),
                        stability_scores=cand["stability"][b].index_select(0, ci), boxes=boxes[b, :k].long(),
                        points=cand["points"][b].index_select(0, ci // cand["n_out"]),
                        candidates=idx_host[b, :k].clone(), rle=rle[b], size=cand["sizes"][b]))
        if polygons:
            out[-1]["polygons"] = polys[b]
    if min_area <= 0 or K == 0:
        return out
    rows_d, cnt, rows_h = _nms(unchanged, valid, boxes, nms_thr)
    for b, r in enumerate(out):
        rows, rh = rows_d[b, :cnt[b]], rows_h[b, :cnt[b]]
        r.update(scores=r["scores"].index_select(0, rows), stability_scores=r["stability_scores"].index_select(0, rows),
                 boxes=boxes[b].index_select(0, rows).long(), points=r["points"].index_select(0, rows),
                 candidates=r["candidates"][rh], rle=[r["rle"][i] for i in rh.tolist()])
        if polygons:
            r["polygons"] = [r["polygons"][i] for i in rh.tolist()]
    return out


def _device_scene(scene: torch.Tensor, dev) -> torch.Tensor:
    """The scene [3, H, W] on dev, copied once in its own memory order (a permuted HWC array stays HWC)."""
    if scene.device == dev:
        return scene
    hwc = scene.permute(1, 2, 0)
    if hwc.is_contiguous():
        return hwc.pin_memory().to(dev, non_blocking=True).permute(2, 0, 1)
    return scene.contiguous().pin_memory().to(dev, non_blocking=True)


def _free_bytes(dev) -> int:
    free, _ = torch.cuda.mem_get_info(dev)
    return free + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)


@torch.no_grad()
def generate_scene_masks(model, scene, *, patch_size: int | None = None, overlap_ratio: float = 0.25,
                         batch_size: int = 4, points_per_side: int = 32, points_per_batch: int = 64,
                         pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95,
                         stability_score_offset: float = 1.0, mask_threshold: float = 0.0,
                         crops_nms_thresh: float = 0.7, crops_n_layers: int = 0, max_hole_area=None,
                         max_sprinkle_area=None, min_mask_region_area: float = 0,
                         coarse_patch_sizes: tuple = (), output_polygons: bool = False) -> dict:
    """Every mask of a whole scene: generate_masks on overlapping windows, merged across windows.

    ``scene``: uint8 RGB [3, H, W] with any strides (a permuted HWC array is fine), on the host or the device; it is
    copied to the device once.  The windows are large_image.slice_origins' P x P windows (P = ``patch_size``, default
    the model's image size; consecutive windows overlap by int(overlap_ratio * P), the last of a row or column is
    shifted inward to end at the scene's edge), each cut to its in-scene part: the crop box (x0, y0, x1, y1) with
    x1 = min(x0 + P, W), y1 = min(y0 + P, H) (``scene_crop_boxes``).

    Each window is exactly ``generate_masks(scene[:, y0:y1, x0:x1], ...)`` with the same parameters, plus the crop-edge
    rule of HF's filter_masks (SAM's _process_batch) after the predicted-IoU and stability filters and before the
    window's NMS: a candidate is dropped when a side of its box, shifted into the scene, lies within 20 px of the crop
    box's side but not within 20 px of the scene's (HF's _is_box_near_crop_edge, fp32).  The survivors of every
    window are shifted into scene coordinates and merged by one box NMS at the same ``crops_nms_thresh``, scored by
    predicted IoU (post_process_for_mask_generation's NMS over every window): a stable descending sort, ties by
    (window in slice order, rank in the window's keep order).  A scene that fits in one window (H <= P and W <= P) is
    generate_masks(scene, output_rle_mask=True): the crop box is the scene, so the rule drops nothing.

    Objects larger than the overlap: as with SAM's crop layers without the whole-image layer, a mask is kept only
    from a window in which its box is more than 20 px from every interior edge.  An object is certain to be found
    only when its extent is below about int(overlap_ratio * P) - 42 px (214 px at the defaults); larger objects
    crossing windows (fields, water bodies) may be found in none, unless a coarse layer finds them.

    ``coarse_patch_sizes`` (P_1 < P_2 < ..., each > P, integers): SAM's crop layers in the other direction, a pyramid
    of coarser windows above the base ones (``scene_layer_windows``).  Layer l is scene_crop_boxes of P_l with the
    same overlap; a size >= max(H, W) is one window, the whole scene, whose edge rule drops nothing.  A layer whose
    windows are those of the previous layer (two sizes that both cover the scene, or a base layer that already is the
    scene) is run once.  Each coarse window runs the same stages, but is resized to the model input by
    ``rsp_resize_aa_pad_u8``, SamImageProcessor's antialiased resize (rsp_resize_pad_u8's cv2 resize aliases at these
    downscales; the base layer keeps it, so its rows do not change).  Each layer's windows are merged as the base
    layer's; then SAM's crop-layer rule prefers the smaller crop: one box NMS at ``crops_nms_thresh`` over [base rows,
    layer 1 rows, ...] ranked by position, so every base row is kept, and a coarse row is kept iff it overlaps no
    earlier kept row above the threshold.  Unlike SAM, whose 1 / crop-area scores tie within a layer, rows of one
    layer are ranked by predicted IoU.  A coarse window's kept masks are pasted, cleaned and encoded in groups of at
    most COARSE_MASK_BYTES.  Every coarse window must have fewer than 2^31 pixels (the mask statistics and RLE
    kernels' limit); invalid sizes raise ValueError before device work.

    Windows run ``batch_size`` at a time through generate_masks' stages: the low-res logits of a batch (805 MB per
    window at the default grid) are freed before the next batch, and the kept masks of each window are encoded as
    COCO RLE of the whole H x W scene straight from the window's bits, which are then freed.  Masks the merge later
    suppresses were encoded for nothing: the price of memory that does not grow with the scene.  Host
    synchronisations: those of generate_masks(output_rle_mask=True) per batch, and one for the merge when some mask
    was kept; with coarse layers, the RLE's two per group of COARSE_MASK_BYTES rather than per batch in them, one
    merge per layer and one for the cross-layer NMS.  More than large_image.MAX_MERGE_CANDIDATES survivors raise ValueError before the merge; a merge
    workspace (N^2 / 8 bytes) or a batch (scene copy, logits, pixel values and the worst case of bits) larger than
    free device memory raises RuntimeError, the batch before any window runs.

    Returns one dict, rows in the merge's keep order, all in scene coordinates:
      rle               COCO compressed RLE dicts {'size': [H, W], 'counts': bytes}
      polygons          with output_polygons: per mask (contours, hierarchy) of the same scene mask as generate_masks
                        gives them, traced with the RLE from the same bits (two more host synchronisations each time)
      scores            fp32 [k] predicted IoU
      stability_scores  fp32 [k]
      boxes             int64 [k, 4] inclusive pixel xyxy
      points            fp32 [k, 2] the prompt of each mask
      tiles             int64 [k] window index in its layer (slice order)
      crop_boxes        int64 [k, 4] xyxy crop box of each mask's window
      layers            int64 [k] 0 for the base layer, l for coarse_patch_sizes[l - 1]
      candidates        int64 [k] (host) candidate index in its window: point * 3 + output mask
      size              (H, W)
    All tensors but ``candidates`` are on the model's device."""
    _check_params(points_per_side, points_per_batch, crops_n_layers, max_hole_area, max_sprinkle_area)
    min_area = _check_region_area(min_mask_region_area)
    if not isinstance(scene, torch.Tensor) or scene.dtype != torch.uint8 or scene.dim() != 3 or scene.shape[0] != 3:
        raise ValueError("the scene must be a uint8 RGB tensor [3, H, W], got "
                         + (f"{scene.dtype} {tuple(scene.shape)}" if isinstance(scene, torch.Tensor)
                            else type(scene).__name__))
    H, W = int(scene.shape[1]), int(scene.shape[2])
    if H < 1 or W < 1:
        raise ValueError(f"the scene is empty: {H} x {W}")
    if patch_size is not None and int(patch_size) < 1:
        raise ValueError(f"patch_size must be >= 1, got {patch_size}")
    if not 0 <= overlap_ratio < 1:
        raise ValueError(f"overlap_ratio must be in [0, 1), got {overlap_ratio}")
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    coarse = _coarse_sizes(coarse_patch_sizes, (H, W))
    if coarse and patch_size is not None and coarse[0] <= int(patch_size):
        raise ValueError(f"coarse_patch_sizes must be greater than the patch size {int(patch_size)}, got {tuple(coarse)}")
    sam = _sam(model)
    dev = sam.prompt_encoder.no_mask_embed.weight.device
    S = sam.varch.image_size
    P = S if patch_size is None else int(patch_size)
    if coarse and coarse[0] <= P:
        raise ValueError(f"coarse_patch_sizes must be greater than the patch size {P}, got {tuple(coarse)}")
    layers = scene_layer_windows((H, W), P, overlap_ratio, coarse)
    p = dict(points_per_side=int(points_per_side), points_per_batch=int(points_per_batch),
             pred_iou_thresh=float(pred_iou_thresh), stability_score_thresh=float(stability_score_thresh),
             stability_score_offset=float(stability_score_offset), mask_threshold=float(mask_threshold))
    nms_thr = float(crops_nms_thresh)

    # what one batch of each layer holds at once, checked before any window runs
    n_cand = 3 * p["points_per_side"] ** 2
    hm = 4 * (S // sam.varch.patch_size)
    free = _free_bytes(dev)
    for l, crops in layers:
        B = min(int(batch_size), len(crops))
        Pl = P if l == 0 else coarse[l - 1]
        ph, pw = min(Pl, H), min(Pl, W)
        bits = B * n_cand * ph * ((pw + 15) // 16 * 2)
        if l:               # one group of masks, and the antialiased resize's horizontal pass
            bits = min(bits, max(COARSE_MASK_BYTES, ph * ((pw + 15) // 16 * 2))) + B * 3 * ph * S
        need = ((0 if scene.device == dev else 3 * H * W) + B * n_cand * hm * hm * 4 + B * 3 * S * S * 4 + bits)
        if need > free:
            raise RuntimeError(f"a {H} x {W} scene in batches of {B} windows of {Pl}^2 needs {need / 2**30:.2f} GiB on "
                               f"{dev} (the scene, {n_cand} candidates' low-res logits per window, the pixel values and "
                               f"the bits if every candidate were kept); {free / 2**30:.2f} GiB are free")

    img = _device_scene(scene, dev)
    merged = []
    for l, crops in layers:
        B = min(int(batch_size), len(crops))
        tiles = []
        for b0 in range(0, len(crops), B):
            boxes_b = crops[b0:b0 + B]
            views = [img[:, y0:y1, x0:x1] for x0, y0, x1, y1 in boxes_b]
            pix, sizes, reshaped = _inputs(sam, views, None, None, None, dev, antialias=l > 0)
            cand = _candidates(sam, sam._encode(pix), sizes, reshaped, p, crops=[(cb, (H, W)) for cb in boxes_b])
            del pix
            idx, counts, idx_host = _nms(cand["iou"], cand["keep"], cand["boxes"], nms_thr)
            places = [(H, W, y0, x0) for x0, y0, _, _ in boxes_b]
            if l:
                out = _coarse_outputs(cand, idx, counts, idx_host, p, S, min_area, nms_thr, places,
                                      polygons=output_polygons)
                del cand, idx
            else:
                out = _outputs(cand, idx, counts, idx_host, p["mask_threshold"], S)
                del cand, idx                                   # the batch's low-res logits
                if min_area > 0:
                    out = _remove_small_regions(out, min_area, nms_thr)
                _add_rle(out, places=places, polygons=output_polygons)
                for r in out:
                    del r["masks"]                              # only the rows and strings stay
            tiles.extend(out)
        merged.append((l, _merge_tiles(tiles, crops, (H, W), nms_thr, dev, output_polygons)))
    if len(merged) == 1:
        res = merged[0][1]
        res["layers"] = torch.zeros(len(res["rle"]), device=dev, dtype=torch.int64)
        return res
    return _merge_layers(merged, nms_thr, dev, output_polygons)


def _check_merge(N: int, what: str, dev) -> None:
    from .large_image import MAX_MERGE_CANDIDATES
    if N > MAX_MERGE_CANDIDATES:
        raise ValueError(f"{what} kept {N} masks; the cross-window merge's dense NMS takes at most "
                         f"{MAX_MERGE_CANDIDATES} candidates")
    ws = N * ((N + 63) // 64) * 8
    free = _free_bytes(dev)
    if ws > free:
        raise RuntimeError(f"the merge of {N} masks from {what} needs a {ws / 2**30:.2f} GiB NMS workspace "
                           f"on {dev}; {free / 2**30:.2f} GiB are free")


def _merge_layers(merged: list, nms_thr: float, dev, polygons: bool = False) -> dict:
    """SAM's crop-layer rule over every layer's merged rows (``merged`` = [(layer, _merge_tiles result)], base first):
    one box NMS over their concatenation ranked by position (equal scores and a stable sort), so a row is dropped only
    by an earlier kept row, of its own layer or a finer one.  One host synchronisation."""
    n = [len(m["rle"]) for _, m in merged]
    N = sum(n)
    _check_merge(N, f"{len(merged)} layers", dev)
    layer_h = torch.repeat_interleave(torch.tensor([l for l, _ in merged]), torch.tensor(n, dtype=torch.int64))
    cat = {key: torch.cat([m[key] for _, m in merged])
           for key in ("scores", "stability_scores", "boxes", "points", "tiles", "crop_boxes", "candidates")}
    res = dict(size=merged[0][1]["size"])
    if polygons:
        res["polygons"] = []
    if N == 0:
        return dict(res, rle=[], layers=layer_h.to(dev), **cat)
    idx, cnt, idx_host = _nms(torch.zeros(1, N, device=dev), torch.ones(1, N, device=dev, dtype=torch.bool),
                              cat["boxes"][None], nms_thr)
    rows, rows_h = idx[0, :cnt[0]], idx_host[0, :cnt[0]]
    rle = [s for _, m in merged for s in m["rle"]]
    res.update({key: v.index_select(0, rows) for key, v in cat.items() if key != "candidates"})
    res.update(rle=[rle[i] for i in rows_h.tolist()], candidates=cat["candidates"][rows_h],
               layers=layer_h[rows_h].pin_memory().to(dev, non_blocking=True))
    if polygons:
        polys = [s for _, m in merged for s in m["polygons"]]
        res["polygons"] = [polys[i] for i in rows_h.tolist()]
    return res


def _merge_tiles(tiles: list, crops: list, hw: tuple, nms_thr: float, dev, polygons: bool = False) -> dict:
    """The cross-window NMS of generate_scene_masks over every window's rows (in slice order, each in keep order)."""
    counts = [r["scores"].shape[0] for r in tiles]
    N = sum(counts)
    _check_merge(N, f"{len(tiles)} windows", dev)
    tile_h = torch.repeat_interleave(torch.arange(len(tiles)), torch.tensor(counts, dtype=torch.int64))
    crop_h = torch.tensor(crops, dtype=torch.int64).view(-1, 4)[tile_h]
    res = dict(rle=[], scores=torch.zeros(0, device=dev), stability_scores=torch.zeros(0, device=dev),
               boxes=torch.zeros(0, 4, device=dev, dtype=torch.int64), points=torch.zeros(0, 2, device=dev),
               tiles=torch.zeros(0, device=dev, dtype=torch.int64),
               crop_boxes=torch.zeros(0, 4, device=dev, dtype=torch.int64),
               candidates=torch.zeros(0, dtype=torch.int64), size=(int(hw[0]), int(hw[1])))
    if polygons:
        res["polygons"] = []
    if N == 0:
        return res
    crop_d = crop_h.pin_memory().to(dev, non_blocking=True)
    off = crop_h[:, [0, 1, 0, 1]].pin_memory().to(dev, non_blocking=True)     # indexed on the host: no sync
    scores = torch.cat([r["scores"] for r in tiles])
    boxes = torch.cat([r["boxes"] for r in tiles]) + off
    points = torch.cat([r["points"] for r in tiles]) + off[:, :2].float()
    idx, cnt, idx_host = _nms(scores[None], torch.ones(1, N, device=dev, dtype=torch.bool), boxes[None], nms_thr)
    k = cnt[0]
    rows, rows_h = idx[0, :k], idx_host[0, :k]
    rle = [s for r in tiles for s in r["rle"]]
    res.update(rle=[rle[i] for i in rows_h.tolist()], scores=scores.index_select(0, rows),
               stability_scores=torch.cat([r["stability_scores"] for r in tiles]).index_select(0, rows),
               boxes=boxes.index_select(0, rows), points=points.index_select(0, rows),
               tiles=tile_h[rows_h].pin_memory().to(dev, non_blocking=True), crop_boxes=crop_d.index_select(0, rows),
               candidates=torch.cat([r["candidates"] for r in tiles])[rows_h])
    if polygons:
        polys = [s for r in tiles for s in r["polygons"]]
        res["polygons"] = [polys[i] for i in rows_h.tolist()]
    return res


def masks_to_bool(result: dict) -> torch.Tensor:
    """The bit-packed ``masks`` of one generate_masks result -> bool [k, H, W] on the same device."""
    bits = result["masks"]
    H, W = result["size"]
    if bits.shape[0] == 0:
        return torch.zeros(0, H, W, dtype=torch.bool, device=bits.device)
    return _lib.unpack_mask_bits(bits, bits.shape[2] * 8)[..., :W]


def mask_dicts(result: dict) -> list:
    """The result of one image as JSON-ready dicts: COCO RLE ``segmentation`` (needs output_rle_mask=True), xywh
    ``bbox`` from the inclusive box, ``predicted_iou``, ``stability_score``, ``point_coords`` [[x, y]], and for a
    generate_scene_masks result the window's ``crop_box`` (xywh, as SAM's automatic mask generator writes it)."""
    out = []
    crops = result["crop_boxes"].tolist() if "crop_boxes" in result else None
    for i, (rle, (x1, y1, x2, y2), s, st, pt) in enumerate(zip(
            result["rle"], result["boxes"].tolist(), result["scores"].tolist(), result["stability_scores"].tolist(),
            result["points"].tolist())):
        row = dict(segmentation=dict(size=rle["size"], counts=rle["counts"].decode()),
                   bbox=[x1, y1, x2 - x1, y2 - y1], predicted_iou=s, stability_score=st, point_coords=[pt])
        if crops is not None:
            cx0, cy0, cx1, cy1 = crops[i]
            row["crop_box"] = [cx0, cy0, cx1 - cx0, cy1 - cy0]
        out.append(row)
    return out


def main(argv=None):
    """The CLI: the mask dicts (--out-format coco) or the GeoJSON FeatureCollection, also returned."""
    ap = argparse.ArgumentParser(description="Segment everything in one image with SAM (HF mask-generation, one crop "
                                             "layer) and write the masks as COCO RLE; with --patch-size, in a whole "
                                             "scene cut into overlapping windows")
    ap.add_argument("image")
    ap.add_argument("--arch", required=True, choices=["base", "large", "huge"])
    ap.add_argument("--checkpoint", required=True, help="HF SamModel weights (.pth / .bin or .safetensors)")
    ap.add_argument("--points-per-side", type=int, default=32)
    ap.add_argument("--points-per-batch", type=int, default=64)
    ap.add_argument("--pred-iou-thresh", type=float, default=0.88)
    ap.add_argument("--stability-score-thresh", type=float, default=0.95)
    ap.add_argument("--stability-score-offset", type=float, default=1.0)
    ap.add_argument("--mask-threshold", type=float, default=0.0)
    ap.add_argument("--crops-nms-thresh", type=float, default=0.7)
    ap.add_argument("--min-mask-region-area", type=float, default=0.0,
                    help="fill holes and remove islands smaller than this many pixels (SAM's min_mask_region_area)")
    ap.add_argument("--patch-size", type=int, default=None,
                    help="scene mode: segment P x P windows of the image and merge them across windows, masks of the "
                         "whole image (each window is resized to the model size).  A mask is kept only from a window "
                         "where its box is more than 20 px from every interior window edge, so objects wider than "
                         "about int(overlap * P) - 42 px may be missed")
    ap.add_argument("--patch-overlap-ratio", type=float, default=0.25, help="scene mode: window overlap ratio")
    ap.add_argument("--batch-size", type=int, default=4, help="scene mode: windows run at once")
    ap.add_argument("--coarse-patch-sizes", type=int, nargs="+", default=None, metavar="P",
                    help="scene mode: layers of coarser windows of these sizes (increasing, above --patch-size; one "
                         ">= the scene's long side is the whole scene) that find objects larger than the overlap; "
                         "each dict then has the \"layer\" it came from (0 = the --patch-size windows)")
    ap.add_argument("--out", default=None, help="JSON file for the mask dicts (default: stdout)")
    ap.add_argument("--out-format", default="coco", choices=("coco", "geojson"),
                    help="coco: the mask dicts with COCO RLE segmentations; geojson: a FeatureCollection, one Feature "
                         "per mask with its outlines as a MultiPolygon in pixel coordinates")
    args = ap.parse_args(argv)
    if args.coarse_patch_sizes is not None and args.patch_size is None:
        ap.error("--coarse-patch-sizes needs --patch-size (scene mode)")

    import cv2

    from .sam_model import RSSamModel
    model = RSSamModel(f"facebook/sam-vit-{args.arch}", init_cfg=dict(type="Pretrained", checkpoint=args.checkpoint))
    model = model.cuda().eval()
    img = cv2.imread(args.image, cv2.IMREAD_COLOR)
    if img is None:
        raise FileNotFoundError(args.image)
    geo = args.out_format == "geojson"
    kw = dict(points_per_side=args.points_per_side, points_per_batch=args.points_per_batch,
              pred_iou_thresh=args.pred_iou_thresh, stability_score_thresh=args.stability_score_thresh,
              stability_score_offset=args.stability_score_offset, mask_threshold=args.mask_threshold,
              crops_nms_thresh=args.crops_nms_thresh, min_mask_region_area=args.min_mask_region_area)
    if args.patch_size is not None:
        rgb = torch.from_numpy(cv2.cvtColor(img, cv2.COLOR_BGR2RGB)).permute(2, 0, 1)      # [3, H, W] view of HWC
        res = generate_scene_masks(model, rgb, patch_size=args.patch_size, overlap_ratio=args.patch_overlap_ratio,
                                   batch_size=args.batch_size, coarse_patch_sizes=tuple(args.coarse_patch_sizes or ()),
                                   output_polygons=geo, **kw)
    else:
        rgb = torch.from_numpy(img).permute(2, 0, 1).flip(0)                 # BGR HWC -> RGB [3, H, W] view
        res = generate_masks(model, rgb.contiguous(), output_rle_mask=True, output_polygons=geo, **kw)[0]
    rows = mask_dicts(res)
    if args.coarse_patch_sizes is not None:
        for row, layer in zip(rows, res["layers"].tolist()):
            row["layer"] = layer
    if geo:
        rows = feature_collection([{k: v for k, v in r.items() if k != "segmentation"} for r in rows], res["polygons"])
    text = json.dumps(rows)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    else:
        print(text)
    return rows


if __name__ == "__main__":
    main()
