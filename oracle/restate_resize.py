"""The test pipeline's keep-ratio Resize + Pad + DetDataPreprocessor restated in float64 numpy (rules 1-5), the
yardstick of rsp_resize_pad_u8 and DetDataPreprocessor(device_transforms=...).

Every RSPrompter / SAM-seg config runs (configs/rsprompter/_base_/rsprompter_anchor.py, rsprompter_query.py,
samseg-maskrcnn.py, samseg-mask2former.py and the -peft-512 configs):

    LoadImageFromFile(to_float32=True) -> Resize(scale=crop_size, keep_ratio=True)
    -> Pad(size=crop_size, pad_val=dict(img=(0.406 * 255, 0.456 * 255, 0.485 * 255), masks=0)) -> PackDetInputs

1. size: mmcv/image/geometric.py rescale_size + _scale_size (with the + 0.5; the reference's own copy in
   mmdet/datasets/transforms/transforms.py:62-98 drops it and only FixScaleResize uses that copy, see :92).
2. resample: cv2.resize(img.astype(float32), (new_w, new_h), INTER_LINEAR) (imgproc/src/resize.cpp resizeGeneric:
   fx = (float)((dx + 0.5) * scale_x - 0.5) in double, sx = floor(fx), fx -= sx, borders clamped to (0, 0) /
   (old - 1, 0); HResizeLinear then VResizeLinear).
3. pad bottom / right with the raw pad_val (mmcv/transforms/processing.py Pad.transform).
4. metainfo: ori_shape = (h, w), scale_factor = (new_w / w, new_h / h) (mmcv Resize._resize_img), img_shape = the
   padded size (Pad overwrites it: "Modified Keys: img, img_shape", mmdet transforms.py:719-724).
5. DetDataPreprocessor (data_preprocessor.py:110-148): BGR -> RGB, (x - mean) / std.

Here the arithmetic is float64 throughout except the coefficients, which are rounded to float exactly as cv2
rounds them; the device kernel computes the interpolation in fp32, so the two differ by fp32 rounding only."""
from __future__ import annotations

import numpy as np


def rescale_size(hw, scale) -> tuple:
    """Rule 1: (h, w) -> (new_h, new_w) for Resize(scale, keep_ratio=True); scale is mmcv's (w, h) pair (only its
    larger and smaller edge matter)."""
    h, w = int(hw[0]), int(hw[1])
    long_edge, short_edge = max(scale), min(scale)
    s = min(long_edge / max(h, w), short_edge / min(h, w))
    return int(h * float(s) + 0.5), int(w * float(s) + 0.5)


def linear_taps(n_old: int, n_new: int):
    """cv2 INTER_LINEAR taps along one axis -> (i int64 [n_new], a float64 [n_new] (the float32 weight))."""
    scale = 1.0 / (n_new / n_old)
    d = np.arange(n_new, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    a = (f - i.astype(np.float32)).astype(np.float32)
    lo = i < 0
    i[lo], a[lo] = 0, 0
    hi = i >= n_old - 1
    i[hi], a[hi] = n_old - 1, 0
    return i, a.astype(np.float64)


def resample(img: np.ndarray, new_hw) -> np.ndarray:
    """Rule 2: [h, w, C] (any real dtype) -> float64 [new_h, new_w, C]; horizontal pass first, then vertical."""
    x = np.asarray(img, dtype=np.float64)
    h, w = x.shape[:2]
    nh, nw = int(new_hw[0]), int(new_hw[1])
    ix, ax = linear_taps(w, nw)
    iy, ay = linear_taps(h, nh)
    ix1, iy1 = np.minimum(ix + 1, w - 1), np.minimum(iy + 1, h - 1)
    ax, ay = ax[None, :, None], ay[:, None, None]
    rows = x[:, ix] * (1 - ax) + x[:, ix1] * ax
    return rows[iy] * (1 - ay) + rows[iy1] * ay


def resize_pad(img: np.ndarray, scale, size, pad_val):
    """Rules 1-4 for one uint8 [h, w, 3] BGR image: -> (float64 [Hp, Wp, 3] BGR, metainfo dict).  size = Pad's
    (w, h); pad_val = 3 raw values (BGR) or one number."""
    h, w = img.shape[:2]
    nh, nw = rescale_size((h, w), scale)
    Wp, Hp = int(size[0]), int(size[1])
    pv = np.broadcast_to(np.asarray(pad_val, dtype=np.float64), (3,))
    out = np.empty((Hp, Wp, 3), dtype=np.float64)
    out[...] = pv
    out[:nh, :nw] = resample(img, (nh, nw))
    meta = dict(ori_shape=(h, w), img_shape=(Hp, Wp), scale_factor=(nw / w, nh / h))
    return out, meta


def pipeline(imgs: list, scale, size, pad_val, mean, std, bgr_to_rgb: bool = True):
    """Rules 1-5 for a batch of uint8 [h, w, 3] BGR images -> (float64 [B, 3, Hp, Wp], list of metainfo dicts with
    pad_shape and batch_input_shape as DetDataPreprocessor writes them)."""
    outs, metas = [], []
    for img in imgs:
        x, meta = resize_pad(img, scale, size, pad_val)
        if bgr_to_rgb:
            x = x[..., ::-1]
        x = (x - np.asarray(mean, dtype=np.float64)) / np.asarray(std, dtype=np.float64)
        outs.append(x.transpose(2, 0, 1))
        meta.update(pad_shape=meta["img_shape"], batch_input_shape=meta["img_shape"])
        metas.append(meta)
    return np.stack(outs), metas
