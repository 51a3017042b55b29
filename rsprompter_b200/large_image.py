"""Whole remote-sensing scenes through the detectors: sliced inference, a cross-tile merge and scene-size RLE masks.

The counterpart of the reference's large-image demo (demo/large_image_demo.py:141-262 over
mmdet/utils/large_image.py:27-104): the scene is cut into overlapping model-size windows (sahi ``slice_image`` with
``auto_slice_resolution=False``), every window is detected, the results are shifted into scene coordinates and
merged with one class-aware NMS (``merge_results_by_nms``).  Here all of it stays on the device:

  * tiles are copied out of the scene in batches and normalised by the detector's own DetDataPreprocessor path
    (the fused uint8 patch-embed loader, or ``rsp_preprocess_u8`` for tiles that overhang a scene smaller than
    the patch, padded with 0 after normalisation as BatchFixedSizePad pads); with an explicit patch size
    (the demo's ``--patch-size``) every window is resized to the model size by ``rsp_resize_pad_u8`` straight
    from the scene, as the test pipeline's keep-ratio Resize + Pad does;
  * every batch leaves ``predict_records`` as one ResultRecord, resident until the merge;
  * the merge is ``rsp_nms_batched`` + ``rsp_compact_keep`` over every valid slot of every tile (mmcv
    ``batched_nms`` semantics, label offset included), or ``rsp_soft_nms_batched`` with ``merge_nms_type='soft_nms'``
    (the demo's ``--merge-nms-type``), or greedy non-maximum merging with ``merge_nms_type='greedy_nmm'`` (sahi's
    GREEDYNMM postprocess, ``rsp_nmm_batched``): an object cut by a tile seam comes out as one instance with the
    union of its fragments' boxes and masks;
  * the kept masks are encoded as COCO RLE of the whole scene by ``rsp_mask_rle_placed_*`` (``rsp_mask_rle_union_*``
    for merged groups) straight from the records' bits: the full-scene bool mask sahi's ``shift_masks`` builds for
    every instance never exists.

The merge's hard NMS and greedy merging are dense: at most 393 216 candidates (tiles x slots), with an n^2 / 8-byte
workspace.  The soft merge takes the same number of candidates with an O(n) workspace.

``python -m rsprompter_b200.large_image CONFIG IMAGE`` writes the COCO result dicts of one scene."""
from __future__ import annotations

import argparse
import json
import math

import torch

from . import _lib
from .detectors import RSPrompterAnchor, RSPrompterQuery, SAMSegMaskRCNN
from .geojson import feature_collection
from .registry import DetDataSample, InstanceData
from .results import ResultRecord, _align16

# rsp_nms_batched keeps one 64-candidate word per candidate and word column in shared memory (48 KB)
MAX_MERGE_CANDIDATES = 48 * 1024 // 8 * 64


def slice_origins(hw: tuple, patch: int, overlap_ratio: float) -> list:
    """Top-left corners (x0, y0) of the patch x patch windows sahi's slice_image(..., auto_slice_resolution=False)
    cuts from an H x W scene, row-major.  Windows step by patch - int(overlap_ratio * patch); the last one of a row
    or column is shifted inward to end at the scene's edge, so a window overhangs the scene only where the scene is
    smaller than the patch."""
    H, W = int(hw[0]), int(hw[1])
    patch = int(patch)
    ov = int(overlap_ratio * patch)
    out = []
    y_min = y_max = 0
    while y_max < H:
        x_min = x_max = 0
        y_max = y_min + patch
        while x_max < W:
            x_max = x_min + patch
            if y_max > H or x_max > W:
                out.append((max(0, min(W, x_max) - patch), max(0, min(H, y_max) - patch)))
            else:
                out.append((x_min, y_min))
            x_min = x_max - ov
        y_min = y_max - ov
    return out


MERGE_NMS_TYPES = ("nms", "soft_nms", "greedy_nmm")
MATCH_METRICS = ("ios", "iou")


def _check_merge_args(nms_type: str, match_metric: str) -> None:
    if nms_type not in MERGE_NMS_TYPES:
        raise ValueError(f"merge nms type {nms_type!r} is not supported (supported: {', '.join(MERGE_NMS_TYPES)})")
    if nms_type == "greedy_nmm" and match_metric not in MATCH_METRICS:
        raise ValueError(f"match metric {match_metric!r} is not supported (supported: {', '.join(MATCH_METRICS)})")


def merge_tile_records(records: list, origins: list, scene_hw: tuple, merge_iou_thr: float = 0.25,
                       score_thr: float = 0.0, window: tuple | None = None, nms_type: str = "nms",
                       match_metric: str = "ios") -> dict:
    """Class-aware NMS of every valid slot of every tile, in scene coordinates.

    ``records`` are ResultRecords of tiles (one image per tile; records of one call share slots and device) and
    ``origins[r]`` lists the (x0, y0) of the first len(origins[r]) images of record r; later images are ignored (the
    padding of a last partial batch).  Each box is shifted by its tile's origin (the fp32 add of sahi's
    shift_bboxes) and clipped to the tile's window intersected with the scene, a no-op for a box inside its tile.
    The candidates are sorted by score, ties by (tile, slot), and merged as mmcv batched_nms(boxes, scores, labels,
    iou_threshold=merge_iou_thr).  Candidates below ``score_thr`` are dropped first; greedy NMS lets a box suppress
    only lower-scored boxes, so that is exactly the unfiltered result restricted to score >= score_thr.  ``window``
    (h, w) is the tile size when it differs from the records' canvas (resized patches: the canvas width is rounded
    up to 16).

    ``nms_type='soft_nms'`` merges as mmcv batched_nms(..., dict(type='soft_nms', iou_threshold=merge_iou_thr)) with
    soft_nms's defaults (sigma 0.5, min_score 1e-3, linear), on the valid slots in (tile, slot) order, which is the
    order InstanceData.cat leaves them in and the tie-break of soft-NMS.  As the reference's merge_results_by_nms does
    (``_, keeps = batched_nms(...)``), the kept rows keep their original scores, in keep order: selection order below
    10 000 candidates, by decayed score at or above it.  ``score_thr`` then drops kept rows scored below it.  Filtering
    before a soft merge would not be the same: a low-scored box can be selected early and decay others.

    ``nms_type='greedy_nmm'`` merges instead of suppressing, as sahi's GREEDYNMM postprocess does: candidates (filtered
    and sorted as for nms) match when their labels are equal and their ``match_metric`` ('ios': intersection over the
    smaller area, or 'iou') is >= merge_iou_thr, in fp32 on the scene boxes.  Walking the sorted candidates, one that no
    earlier keeper absorbed becomes a keeper and absorbs every later unabsorbed candidate it matches, so the keepers
    are exactly nms's kept rows and each other candidate joins the first keeper in order that matches it (no
    transitivity: what a member matches is not absorbed through it).  A keeper's row has the element-wise union of its
    members' boxes, its own score and label; its mask is the OR of its members' masks.  Unlike sahi's loop, a member
    is not tested again against the growing merged box: every matched member joins its group.  The result also has
    members int64 [m, 3] (record, image, slot) and member_offsets int64 [k + 1] on the host: group i is
    members[member_offsets[i]:member_offsets[i + 1]], its keeper first, then its absorbed members in sort order.

    Returns dict(bboxes fp32 [k, 4], scores [k], labels int64 [k] on the device, in descending score order (soft: keep
    order), and source int64 [k, 3] on the host: (record, image, slot) of each kept row).  One host synchronisation
    (two for soft_nms: the number of label groups is read first)."""
    _check_merge_args(nms_type, match_metric)
    H, W = int(scene_hw[0]), int(scene_hw[1])
    assert len(records) == len(origins) and records, "one origin list per record"
    M = records[0].slots
    rows, counts, win, src = [], [], [], []
    for r, (rec, org) in enumerate(zip(records, origins)):
        assert rec.slots == M and 0 < len(org) <= rec.batch, "records of one merge share their slot count"
        n = len(org)
        rows.append(rec.rows[:n])
        counts.append(rec.counts[:n])
        ph, pw = window or rec.hw
        for b, (x0, y0) in enumerate(org):
            win.append((x0, y0, min(x0 + pw, W), min(y0 + ph, H)))
            src.append((r, b))
    T = len(src)
    N = T * M
    if N > MAX_MERGE_CANDIDATES:
        raise ValueError(f"{T} tiles x {M} slots = {N} merge candidates; the dense NMS takes at most "
                         f"{MAX_MERGE_CANDIDATES}")
    rows = torch.cat(rows)                                        # [T, M, 6]
    counts = torch.cat(counts)
    dev = rows.device
    win = torch.tensor(win, dtype=torch.float32).pin_memory().to(dev, non_blocking=True)
    lo, hi = win[:, None, [0, 1, 0, 1]], win[:, None, [2, 3, 2, 3]]
    boxes = torch.minimum(torch.maximum(rows[..., :4] + lo, lo), hi)
    scores = rows[..., 4]
    valid = torch.arange(M, device=dev)[None, :] < counts[:, None]
    src = torch.tensor(src, dtype=torch.int64).view(-1, 2)
    if nms_type == "soft_nms":
        return _soft_merge(boxes.reshape(N, 4), scores.reshape(N), rows[..., 5].reshape(N).long(), valid.reshape(N),
                           merge_iou_thr, score_thr, src, M)
    if score_thr > 0:
        valid &= scores >= score_thr
    key = torch.where(valid, scores, torch.full_like(scores, -math.inf)).reshape(N)
    _, order = torch.sort(key, descending=True, stable=True)     # invalid slots last; ties by (tile, slot)
    nvalid = valid.sum().to(torch.int32).view(1)
    boxes_s = boxes.reshape(N, 4)[order].contiguous()
    scores_s = scores.reshape(N)[order].contiguous()
    labels_s = rows[..., 5].reshape(N)[order].long().contiguous()
    if nms_type == "greedy_nmm":
        return _nmm_merge(boxes_s, scores_s, labels_s, nvalid, order, merge_iou_thr, match_metric, src, M)
    keep = _lib.nms_batched(boxes_s[None], labels_s[None], nvalid, merge_iou_thr)
    ob, os_, ol, oi, cnt = _lib.compact_keep(keep, boxes_s[None], scores_s[None], labels_s[None], N)
    flat = order[oi[0].clamp(min=0).long()]
    host = torch.cat([cnt.long(), flat]).cpu()                   # the one host sync: count + sources
    k = int(host[0])
    flat = host[1:1 + k]
    tile, slot = flat // M, flat % M
    return dict(bboxes=ob[0, :k], scores=os_[0, :k], labels=ol[0, :k],
                source=torch.cat([src[tile], slot[:, None]], dim=1))


def _soft_merge(boxes, scores, labels, valid, iou_thr, score_thr, src, M) -> dict:
    """The soft_nms branch of merge_tile_records over the N = tiles x slots candidates (flat, valid flags)."""
    _, order = torch.sort((~valid).to(torch.uint8), stable=True)       # valid slots first, (tile, slot) order kept
    nvalid = valid.sum().to(torch.int32).view(1)
    b = boxes[order].contiguous()
    lab = labels[order].contiguous()
    groups = int(torch.where(valid, labels, torch.zeros_like(labels)).max()) + 1   # host sync 1: label groups
    if groups > 1024:
        raise ValueError(f"soft-NMS merge takes labels below 1024, got {groups - 1}")
    ob, _, ol, oi, cnt = _lib.soft_nms_batched(b[None], scores[order].contiguous()[None], lab[None], nvalid, groups,
                                               iou_thr)
    flat_d = order[oi[0].clamp(min=0).long()]
    os_ = scores[flat_d]                                               # the kept rows' original scores
    n = int(boxes.shape[0])
    keep = (torch.arange(n, device=boxes.device) < cnt[0]) & (os_ >= score_thr)
    host = torch.cat([keep.long(), flat_d]).cpu()                       # host sync 2: kept rows + sources
    sel = host[:n].bool()
    idx = torch.nonzero(sel).view(-1)
    flat = host[n:][sel]
    tile, slot = flat // M, flat % M
    idx_d = idx.to(boxes.device, non_blocking=True)
    return dict(bboxes=ob[0, idx_d], scores=os_[idx_d], labels=ol[0, idx_d],
                source=torch.cat([src[tile], slot[:, None]], dim=1))


def _nmm_merge(boxes_s, scores_s, labels_s, nvalid, order, thr, metric, src, M) -> dict:
    """The greedy_nmm branch of merge_tile_records over the N sorted candidates (valid prefix of nvalid)."""
    N = int(boxes_s.shape[0])
    dev = boxes_s.device
    keep, owner = _lib.nmm_batched(boxes_s[None], labels_s[None], nvalid, thr, metric)
    pos = torch.arange(N, device=dev)
    grp = torch.where(keep[0].bool(), pos, owner[0].long())          # each valid candidate's keeper, -1 invalid
    member = grp >= 0
    idx = grp.clamp(min=0)[:, None].expand(N, 2)
    lo = boxes_s[:, :2].scatter_reduce(0, idx, torch.where(member[:, None], boxes_s[:, :2], math.inf), "amin")
    hi = boxes_s[:, 2:].scatter_reduce(0, idx, torch.where(member[:, None], boxes_s[:, 2:], -math.inf), "amax")
    merged = torch.cat([lo, hi], dim=1).contiguous()
    ob, os_, ol, oi, cnt = _lib.compact_keep(keep, merged[None], scores_s[None], labels_s[None], N)
    # members grouped by keeper in keeper order; a keeper precedes what it absorbed, so the stable sort puts it first
    gkey, morder = torch.sort(torch.where(member, grp, N), stable=True)
    kpos = oi[0].long().clamp(min=0)
    starts = torch.searchsorted(gkey, kpos)
    host = torch.cat([cnt.long(), nvalid.long(), order[kpos], starts, order[morder]]).cpu()   # the one host sync
    k, m = int(host[0]), int(host[1])
    flat = host[2:2 + k]
    offsets = torch.cat([host[2 + N:2 + N + k], torch.tensor([m])])
    mflat = host[2 + 2 * N:2 + 2 * N + m]
    return dict(bboxes=ob[0, :k], scores=os_[0, :k], labels=ol[0, :k],
                source=torch.cat([src[flat // M], (flat % M)[:, None]], dim=1),
                members=torch.cat([src[mflat // M], (mflat % M)[:, None]], dim=1), member_offsets=offsets)


def _slots(model) -> int:
    if isinstance(model, RSPrompterQuery):
        return int(model.test_cfg.get("max_per_image", 100))
    return int(model.test_cfg.rcnn.get("max_per_img", 100))


def _record_nbytes(B: int, M: int, hw: tuple) -> int:
    return _align16(B * M * hw[0] * (hw[1] // 8)) + _align16(B * M * 24) + _align16(B * 4)


@torch.no_grad()
def predict_large_image(model, image, overlap_ratio: float = 0.25, merge_iou_thr: float = 0.25,
                        score_thr: float = 0.0, batch_size: int = 8, patch_size: int | None = None,
                        merge_nms_type: str = "nms", merge_match_metric: str = "ios",
                        output_polygons: bool = False) -> DetDataSample:
    """Detect a whole scene: slice, run the tiles in batches, merge across tiles, encode the kept masks.

    ``image`` is the scene as mmcv.imread decodes it, uint8 [H, W, 3] BGR: a numpy array or a tensor on the host
    (copied to the device once, pinned) or on the model's device.  With ``patch_size=None`` tiles are model-size
    (``image_size``) windows, never resized.  An explicit ``patch_size`` P cuts P x P windows and resizes each (its
    in-scene part when the scene is smaller than P) to the model size the way the test pipeline's keep-ratio Resize
    + Pad does (the reference demo's ``--patch-size``, whose inference_detector runs every slice through that
    pipeline); P = image_size on a scene at least that large is the unresized path.  The last partial batch repeats
    a tile whose slots are ignored, so every batch has one shape and enable_cuda_graphs() replays one graph.  No
    host synchronisation happens per tile or per batch; the merge reads the kept rows once and the RLE encode
    synchronises twice.

    ``merge_nms_type`` ('nms' or 'soft_nms', the demo's ``--merge-nms-type``, or 'greedy_nmm') selects the cross-tile
    merge; see merge_tile_records for what soft_nms returns and how ``score_thr`` applies to it.  'greedy_nmm' joins
    matching rows (``merge_match_metric`` 'ios' or 'iou' >= merge_iou_thr) into one instance with the union box and
    the union mask of its members.

    Returns a DetDataSample with ori_shape = img_shape = (H, W), scale_factor (1, 1) and pred_instances: bboxes,
    scores, labels on the device in descending score order, masks a list of {'size': [H, W], 'counts': bytes} (the
    test_cfg.rle_masks convention, passed through by CocoMetric.process).  ``output_polygons`` adds
    pred_instances.polygons: per mask, mask_polygons' (contours, hierarchy) of the same scene mask, in scene pixel
    coordinates (two more host synchronisations)."""
    _check_merge_args(merge_nms_type, merge_match_metric)
    records, batches = run_tiles(model, image, overlap_ratio, batch_size, patch_size=patch_size,
                                 merge_nms_type=merge_nms_type)
    H, W = int(image.shape[0]), int(image.shape[1])
    window = None if patch_size is None else (int(patch_size), int(patch_size))
    merged = merge_tile_records(records, batches, (H, W), merge_iou_thr=merge_iou_thr, score_thr=score_thr,
                                window=window, nms_type=merge_nms_type, match_metric=merge_match_metric)
    if merge_nms_type == "greedy_nmm":
        canvases = _merged_canvases(records, batches, merged["members"], merged["member_offsets"], (H, W), window)
        masks = _merged_rle(records, canvases)
    else:
        canvases = _kept_canvases(records, batches, merged["source"], (H, W), window)
        masks = _kept_rle(records, canvases)
    ds = DetDataSample(metainfo=dict(ori_shape=(H, W), img_shape=(H, W), scale_factor=(1.0, 1.0)))
    ds.pred_instances = InstanceData(bboxes=merged["bboxes"], scores=merged["scores"], labels=merged["labels"],
                                     masks=masks)
    if output_polygons:
        ds.pred_instances.polygons = mask_polygons(records, canvases)
    return ds


@torch.no_grad()
def run_tiles(model, image, overlap_ratio: float = 0.25, batch_size: int = 8, patch_size: int | None = None,
              merge_nms_type: str = "nms"):
    """The tile stage of predict_large_image -> (records, origins per record), everything left on the device.
    Records of resized patches hold each tile's result in P x P window coordinates on a canvas of
    (P, P rounded up to 16)."""
    if not isinstance(model, (RSPrompterAnchor, RSPrompterQuery, SAMSegMaskRCNN)):
        raise NotImplementedError(f"large-scene inference needs a detector with per-tile result records "
                                  f"(RSPrompterAnchor, RSPrompterQuery, SAMSegMaskRCNN), not {type(model).__name__}")
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    dev = next(model.parameters()).device
    img = torch.from_numpy(image) if not isinstance(image, torch.Tensor) else image
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError(f"the scene must be uint8 [H, W, 3] (BGR, as mmcv.imread decodes it), got "
                         f"{img.dtype} {tuple(img.shape)}")
    H, W = int(img.shape[0]), int(img.shape[1])
    S = int(model.backbone.vision_encoder.arch.image_size)
    P = S if patch_size is None else int(patch_size)
    if P < 1:
        raise ValueError("patch_size must be >= 1")
    resize = patch_size is not None and (P != S or H < P or W < P)
    origins = slice_origins((H, W), P, overlap_ratio)
    B = min(batch_size, len(origins))
    batches = [origins[i:i + B] for i in range(0, len(origins), B)]
    M = _slots(model)
    rec_hw = (P, (P + 15) // 16 * 16) if resize else (P, P)

    # everything that stays resident until the merge, checked before any tile runs
    N = len(origins) * M
    if N > MAX_MERGE_CANDIDATES:
        raise ValueError(f"{len(origins)} tiles x {M} slots = {N} merge candidates; the dense NMS takes at most "
                         f"{MAX_MERGE_CANDIDATES}")
    merge_ws = (_lib.soft_nms_workspace_bytes(1, N, 1024) + N * 64 if merge_nms_type == "soft_nms"   # O(N) + gathers
                else N * ((N + 63) // 64) * 8 + (N * 4 if merge_nms_type == "greedy_nmm" else 0))   # + owner
    need = (len(batches) * _record_nbytes(B, M, rec_hw) + (0 if img.is_cuda else H * W * 3)
            + merge_ws + (B * 3 * S * S * 4 if resize else 0))
    free, _ = torch.cuda.mem_get_info(dev)
    free += torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    if need > free:
        raise RuntimeError(f"a {H} x {W} scene needs {need / 2**30:.2f} GiB resident on {dev} ({len(origins)} tiles "
                           f"of {P}^2 in {len(batches)} result records, the scene and the merge workspace); "
                           f"{free / 2**30:.2f} GiB are free")

    scene = img.to(dev) if img.is_cuda else img.pin_memory().to(dev, non_blocking=True)
    dp = model.data_preprocessor
    mean, std, swap = dp._norm3() if dp is not None else ((0.0,) * 3, (1.0,) * 3, False)
    if resize:
        return _run_resized_tiles(model, scene, batches, B, M, S, P, rec_hw, (mean, std, swap)), batches
    overhang = H < P or W < P
    if overhang:    # every window overhangs: normalised fp32 tiles padded with 0, clipped to their in-scene extent
        buf = torch.empty(B, 3, P, P, dtype=torch.float32, device=dev)
        hv, wv = min(P, H), min(P, W)
        shapes = torch.tensor([[hv, wv]] * B, dtype=torch.float32).pin_memory().to(dev, non_blocking=True)
    else:           # uint8 HWC tiles: the normalisation is fused into the patch-embed loader
        buf = torch.empty(B, P, P, 3, dtype=torch.uint8, device=dev)
    records = []
    for org in batches:
        tiles = org + [org[-1]] * (B - len(org))
        for i, (x0, y0) in enumerate(tiles):
            view = scene[y0:y0 + P, x0:x0 + P]
            if overhang:
                _lib.preprocess_u8(view.permute(2, 0, 1), buf[i], mean, std, swap, 0.0)
            else:
                buf[i].copy_(view)
        if overhang:
            batch = buf
            batch.rsp_img_shapes = shapes
        else:
            batch = buf.permute(0, 3, 1, 2)
            batch.rsp_norm = (mean, std, swap)
        records.append(model.predict_records(batch, record=ResultRecord(B, M, (P, P), device=dev)))
    return records, batches


def _run_resized_tiles(model, scene, batches, B, M, S, P, rec_hw, norm):
    """Tiles of P x P resized to the model size S by rsp_resize_pad_u8 straight from the device scene (one launch per
    batch), then predict_records with the samples Resize + Pad would write: records in window coordinates."""
    from .preprocess import rescale_size, resize_metainfo
    H, W = int(scene.shape[0]), int(scene.shape[1])
    hv, wv = min(P, H), min(P, W)                  # a window's in-scene part (sahi slices it so)
    new_hw = rescale_size((hv, wv), (S, S))
    meta = dict(resize_metainfo((hv, wv), new_hw, (S, S)), batch_input_shape=(S, S), pad_shape=(S, S))
    samples = [DetDataSample(metainfo=dict(meta)) for _ in range(B)]
    mean, std, swap = norm
    pad = tuple(reversed(mean)) if swap else tuple(mean)    # the configs pad with the mean: 0 after normalisation
    buf = torch.empty(B, 3, S, S, dtype=torch.float32, device=scene.device)
    records = []
    for org in batches:
        tiles = org + [org[-1]] * (B - len(org))
        views = [scene[y0:y0 + hv, x0:x0 + wv].permute(2, 0, 1) for x0, y0 in tiles]
        _lib.resize_pad_u8(views, [new_hw] * B, buf, mean, std, swap, pad)
        records.append(model.predict_records(buf, record=ResultRecord(B, M, rec_hw, device=scene.device),
                                             batch_data_samples=samples))
    return records


def _kept_canvases(records: list, origins: list, source: torch.Tensor, scene_hw: tuple, window: tuple | None) -> list:
    """Union-mode canvases of the kept masks (``source`` rows (record, image, slot)), one part each: the record's mask
    placed at its tile origin in the H x W scene, cut to its tile window."""
    H, W = int(scene_hw[0]), int(scene_hw[1])
    return [(H, W, [_part(records, origins, r, b, s, H, W, window)]) for r, b, s in source.tolist()]


def _merged_canvases(records: list, origins: list, members: torch.Tensor, member_offsets: torch.Tensor,
                     scene_hw: tuple, window: tuple | None) -> list:
    """Union-mode canvases of greedy_nmm's merged rows: row i's parts are its members'
    members[member_offsets[i]:member_offsets[i + 1]] masks, placed as in _kept_canvases."""
    H, W = int(scene_hw[0]), int(scene_hw[1])
    mem = members.tolist()
    offs = member_offsets.tolist()
    return [(H, W, [_part(records, origins, r, b, s, H, W, window) for r, b, s in mem[offs[i]:offs[i + 1]]])
            for i in range(len(offs) - 1)]


def _part(records: list, origins: list, r: int, b: int, s: int, H: int, W: int, window: tuple | None) -> tuple:
    """(record, byte offset, row bytes, rows, h, w, y0, x0) of slot s of image b of record r in the scene."""
    rec = records[r]
    P, M = rec.hw[0], rec.slots
    ph, pw = window or rec.hw
    ld = rec.hw[1] // 8
    x0, y0 = origins[r][b]
    return (r, (b * M + s) * P * ld, ld, P, min(ph, H - y0), min(pw, W - x0), y0, x0)


def _kept_rle(records: list, canvases: list) -> list:
    groups = [(records[r].buf, [(off, ld, rows, h, w, H, W, y0, x0)])
              for H, W, [(r, off, ld, rows, h, w, y0, x0)] in canvases]
    return [dict(size=[H, W], counts=c) for (H, W, _), c in zip(canvases, _lib.mask_rle_placed(groups, packed=True))]


def _merged_rle(records: list, canvases: list) -> list:
    return [dict(size=[H, W], counts=c) for (H, W, _), c in
            zip(canvases, _lib.mask_rle_union([rec.buf for rec in records], canvases, packed=True))]


def mask_polygons(records: list, canvases: list) -> list:
    """Per canvas (_kept_canvases / _merged_canvases) the (contours, hierarchy) of cv2.findContours(scene mask,
    RETR_CCOMP, CHAIN_APPROX_SIMPLE), traced on the GPU from the records' bits: int32 [k, 2] (x, y) scene pixel
    indices and int32 [1, n, 4] (None for an empty mask); two host synchronisations per workspace-bounded call."""
    return _lib.mask_contours([rec.buf for rec in records], canvases, _lib.CHAIN_APPROX_SIMPLE)


def encode_kept_masks(records: list, origins: list, source: torch.Tensor, scene_hw: tuple,
                      window: tuple | None = None) -> list:
    """COCO RLE dicts of the kept masks (``source`` rows (record, image, slot) from merge_tile_records) as masks of
    the whole H x W scene, encoded from the records' bits; two host synchronisations.  ``window`` as in
    merge_tile_records."""
    return _kept_rle(records, _kept_canvases(records, origins, source, scene_hw, window))


def encode_merged_masks(records: list, origins: list, members: torch.Tensor, member_offsets: torch.Tensor,
                        scene_hw: tuple, window: tuple | None = None) -> list:
    """COCO RLE dicts of greedy_nmm's merged rows: row i is the OR of the masks of members[member_offsets[i]:
    member_offsets[i + 1]] (rows (record, image, slot) from merge_tile_records), each placed in the H x W scene at its
    tile origin and cut to its tile window, encoded by rsp_mask_rle_union_* from the records' bits (a group of one is
    the placed encode's string); two host synchronisations.  ``window`` as in merge_tile_records."""
    return _merged_rle(records, _merged_canvases(records, origins, members, member_offsets, scene_hw, window))


def coco_results(ds: DetDataSample, image_id=0, label_to_cat=None) -> list:
    """COCO result dicts of one scene, as CocoMetric.results2json writes them: xywh bbox, score, category_id and the
    RLE segmentation with ``counts`` as str."""
    p = ds.pred_instances
    out = []
    for (x1, y1, x2, y2), score, label, m in zip(p.bboxes.tolist(), p.scores.tolist(), p.labels.tolist(), p.masks):
        cat = int(label) if label_to_cat is None else label_to_cat[int(label)]
        out.append(dict(image_id=image_id, bbox=[x1, y1, x2 - x1, y2 - y1], score=float(score), category_id=cat,
                        segmentation=dict(size=m["size"], counts=m["counts"].decode())))
    return out


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="Detect one large scene: sliced inference, merge, COCO RLE masks")
    ap.add_argument("config")
    ap.add_argument("image")
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--patch-overlap-ratio", type=float, default=0.25)
    ap.add_argument("--merge-iou-thr", type=float, default=0.25)
    ap.add_argument("--score-thr", type=float, default=0.0)
    ap.add_argument("--merge-nms-type", default="nms", choices=MERGE_NMS_TYPES,
                    help="NMS type of the cross-tile merge (soft_nms: linear, sigma 0.5, min_score 1e-3; greedy_nmm: "
                         "matching rows are merged into one instance with the union box and mask)")
    ap.add_argument("--merge-match-metric", default="ios", choices=MATCH_METRICS,
                    help="match metric of greedy_nmm, compared with --merge-iou-thr (ios: intersection over the "
                         "smaller area)")
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--patch-size", type=int, default=None,
                    help="window size; each window is resized to the model size (default: model-size windows, "
                         "not resized)")
    ap.add_argument("--out", default=None, help="JSON file for the result dicts (default: stdout)")
    ap.add_argument("--out-format", default="coco", choices=("coco", "geojson"),
                    help="coco: COCO result dicts with RLE masks; geojson: a FeatureCollection, one Feature per result "
                         "with the mask's outlines as a MultiPolygon in pixel coordinates")
    return ap


def main(argv=None):
    """The CLI: the result dicts (--out-format coco) or the GeoJSON FeatureCollection, also returned."""
    args = build_parser().parse_args(argv)

    import cv2

    from .registry import MODELS, Config
    cfg = Config.fromfile(args.config)
    model = MODELS.build(cfg.model)
    if args.checkpoint:
        sd = torch.load(args.checkpoint, map_location="cpu")
        model.load_state_dict(sd.get("state_dict", sd), strict=True)
    model = model.cuda().eval()
    img = cv2.imread(args.image, cv2.IMREAD_COLOR)
    if img is None:
        raise FileNotFoundError(args.image)
    ds = predict_large_image(model, img, overlap_ratio=args.patch_overlap_ratio, merge_iou_thr=args.merge_iou_thr,
                             score_thr=args.score_thr, batch_size=args.batch_size, patch_size=args.patch_size,
                             merge_nms_type=args.merge_nms_type, merge_match_metric=args.merge_match_metric,
                             output_polygons=args.out_format == "geojson")
    res = coco_results(ds)
    if args.out_format == "geojson":
        res = feature_collection([{k: v for k, v in r.items() if k != "segmentation"} for r in res],
                                 ds.pred_instances.polygons)
    text = json.dumps(res)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    else:
        print(text)
    return res


if __name__ == "__main__":
    main()
