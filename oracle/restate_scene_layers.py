"""Plain restatement of the coarse layers of segment-everything over a whole scene (TEST INFRASTRUCTURE, see
oracle/__init__.py): torchvision's antialiased uint8 resize in int64 numpy, the windows of each layer, and the
cross-layer merge over restate_scene_mask_generation.merge rows.  rsprompter_b200.mask_generation.generate_scene_masks
(coarse_patch_sizes) and rsp_resize_aa_pad_u8 are checked against it; tests/test_scene_layers_cpu.py pins the resize
to torchvision.transforms.v2.functional.resize(uint8, antialias=True) byte for byte.

Citations: T: = aten/src/ATen/native/cpu/UpSampleKernel.cpp (_compute_index_ranges_weights,
_compute_index_ranges_int16_weights: the separable uint8 path torchvision calls with antialias=True)."""
from __future__ import annotations

import numpy as np
import torch

from . import restate_mask_generation as R
from . import restate_scene_mask_generation as M


def aa_weights(n_in: int, n_out: int) -> tuple:
    """One axis of the bilinear antialiased filter, weights in double then fixed point (T:).
    -> (xmin int [n_out], xsize int [n_out], integer weights int64 [n_out, k], prec)."""
    scale = n_in / n_out
    support = scale if scale >= 1.0 else 1.0
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    xmins, xsizes, rows = [], [], []
    for i in range(n_out):
        center = scale * (i + 0.5)
        xmin = max(int(center - support + 0.5), 0)
        xsize = min(int(center + support + 0.5), n_in) - xmin
        w = [max(0.0, 1.0 - abs((j + xmin - center + 0.5) * inv)) for j in range(xsize)]
        total = 0.0
        for v in w:
            total += v
        xmins.append(xmin)
        xsizes.append(xsize)
        rows.append([v / total for v in w] if total != 0.0 else w)
    k = max(xsizes)
    w_max = max(max(r) for r in rows)
    prec = 0
    while prec < 22 and int(0.5 + w_max * (1 << (prec + 1))) < (1 << 15):
        prec += 1
    wi = np.zeros((n_out, k), np.int64)
    for i, r in enumerate(rows):
        for j, v in enumerate(r):
            wi[i, j] = int(v * (1 << prec) + 0.5)
    return np.array(xmins), np.array(xsizes), wi, prec


def _pass(img: np.ndarray, n_out: int, axis: int) -> np.ndarray:
    """One fixed-point pass along ``axis`` of an int64 array: clamp((2^(prec-1) + sum p * w) >> prec, 0, 255)."""
    n_in = img.shape[axis]
    xmin, xsize, wi, prec = aa_weights(n_in, n_out)
    src = np.moveaxis(img, axis, -1)
    acc = np.zeros(src.shape[:-1] + (n_out,), np.int64)
    for j in range(wi.shape[1]):
        idx = np.minimum(xmin + j, n_in - 1)
        w = np.where(j < xsize, wi[:, j], 0)
        acc += src[..., idx] * w
    out = np.clip((acc + (1 << (prec - 1))) >> prec, 0, 255)
    return np.moveaxis(out, -1, axis)


def resize_aa(img, size: tuple) -> np.ndarray:
    """uint8 [C, H, W] -> uint8 [C, h, w]: the horizontal pass first (to uint8), then the vertical one; an axis whose
    size does not change is not resampled."""
    a = np.asarray(img).astype(np.int64)
    h, w = int(size[0]), int(size[1])
    if a.shape[2] != w:
        a = _pass(a, w, 2)
    if a.shape[1] != h:
        a = _pass(a, h, 1)
    return a.astype(np.uint8)


def layer_windows(hw: tuple, patch: int, overlap_ratio: float, coarse_patch_sizes=()) -> list:
    """The windows of every layer: [(layer, crop boxes)] with layer 0 the base patch, layer l coarse_patch_sizes[l - 1];
    a layer whose windows are those of the previous layer that runs is left out."""
    out = [(0, M.crop_boxes(hw, patch, overlap_ratio))]
    for l, p in enumerate(coarse_patch_sizes, 1):
        boxes = M.crop_boxes(hw, p, overlap_ratio)
        if boxes != out[-1][1]:
            out.append((l, boxes))
    return out


def merge_layers(layers: list, crops_nms_thresh: float) -> dict:
    """SAM's crop-layer rule across layers: ``layers`` = [(layer, merged rows)] with each entry a
    restate_scene_mask_generation.merge result in scene coordinates, base layer first.  One box NMS over the
    concatenation ranked by position, so every base row survives and a coarse row is kept iff it overlaps no earlier
    kept row above the threshold.  -> the merge rows concatenated and selected, plus ``layers``, in keep order."""
    cat = {k: torch.cat([m[k] for _, m in layers]) for k in layers[0][1]}
    cat["layers"] = torch.cat([torch.full((len(m["boxes"]),), l, dtype=torch.int64) for l, m in layers])
    n = len(cat["layers"])
    keep = R.nms(cat["boxes"], torch.zeros(n), crops_nms_thresh)
    return {k: v[keep] for k, v in cat.items()}
