"""DetDataPreprocessor for inference (mmdet/models/data_preprocessors/data_preprocessor.py:29-149 over mmengine's
ImgDataPreprocessor): collate -> BGR->RGB -> float -> (x - mean) / std -> pad bottom/right to a multiple of
``pad_size_divisor`` -> stack, and ``batch_input_shape`` / ``pad_shape`` written into the data samples.

This sits in front of the hot path (SURVEY.md 8(f2)).  uint8 images (what ``PackDetInputs`` emits) are uploaded as
bytes and converted by ``rsp_preprocess_u8`` (channel flip, normalise with true fp32 division, pad) straight into
their slot of the batch tensor - one kernel per image, no CPU arithmetic.  When the consumer is one of this package's
detectors (``fuse_patch_embed=True``) and the images already have the batch shape, the uint8 batch itself is handed
over with the normalisation attached (``tensor.rsp_norm``): ``rsp_patchify16_u8`` then applies it inside the
patch-embed operand loader and the fp32 image never exists.  Float inputs keep the round-1 torch expression.
Training-time batch augmentations (``BatchFixedSizePad`` ...) are ignored: the reference applies them only when
``training=True`` (data_preprocessor.py:145-147).

``device_transforms=[dict(type='Resize', scale=..., keep_ratio=True), dict(type='Pad', size=..., pad_val=...)]``
moves the test pipeline's keep-ratio Resize and Pad here: the two dicts are taken from ``test_pipeline`` unchanged
(and ``to_float32`` dropped from LoadImageFromFile), so the original uint8 bytes of images of any size are uploaded
with one pinned copy and resized, padded, flipped and normalised by one ``rsp_resize_pad_u8`` launch.  The resize is
cv2's float32 INTER_LINEAR (what ``to_float32=True`` pipelines compute); the metainfo is what Resize and Pad write
(``rescale_size`` / ``resize_metainfo`` below, the one place this rule lives)."""
from __future__ import annotations

import math

import torch
from torch import nn

from . import _lib
from .registry import MODELS, BaseModule, DetDataSample


def rescale_size(hw, scale) -> tuple:
    """mmcv rescale_size + _scale_size for Resize(scale, keep_ratio=True): (h, w) -> (new_h, new_w) with
    s = min(max(scale) / max(h, w), min(scale) / min(h, w)) and new = int(old * s + 0.5)."""
    h, w = int(hw[0]), int(hw[1])
    s = min(max(scale) / max(h, w), min(scale) / min(h, w))
    return int(h * float(s) + 0.5), int(w * float(s) + 0.5)


def resize_metainfo(hw, new_hw, pad_hw) -> dict:
    """What Resize + Pad write: ori_shape, scale_factor = (new_w / w, new_h / h) as Python floats, and img_shape = the
    padded size (mmcv Pad overwrites it, mmdet transforms.py:719-724)."""
    h, w = int(hw[0]), int(hw[1])
    return dict(ori_shape=(h, w), scale_factor=(new_hw[1] / w, new_hw[0] / h),
                img_shape=(int(pad_hw[0]), int(pad_hw[1])))


def _parse_device_transforms(cfg, pad_size_divisor: int):
    """-> (scale, (Hp, Wp), raw pad value per input channel) of [Resize(keep_ratio=True), Pad(size=...)]."""
    cfg = [dict(t) for t in cfg]
    kinds = [str(t.get("type", "")).split(".")[-1] for t in cfg]
    if kinds != ["Resize", "Pad"]:
        raise ValueError(f"device_transforms supports exactly [Resize, Pad] (the configs' test pipeline), got {kinds}")
    rs, pd = cfg
    extra = set(rs) - {"type", "scale", "keep_ratio", "backend", "interpolation", "clip_object_border"}
    if extra or rs.get("scale") is None or not rs.get("keep_ratio", False):
        raise ValueError(f"device_transforms Resize needs scale= and keep_ratio=True (no {sorted(extra) or 'other'} "
                         f"options): {rs}")
    if rs.get("interpolation", "bilinear") != "bilinear" or rs.get("backend", "cv2") != "cv2":
        raise ValueError(f"device_transforms Resize reproduces cv2 bilinear only: {rs}")
    scale = rs["scale"]
    scale = (int(scale), int(scale)) if isinstance(scale, (int, float)) else tuple(int(s) for s in scale)
    extra = set(pd) - {"type", "size", "pad_val", "padding_mode"}
    if extra or pd.get("size") is None or pd.get("padding_mode", "constant") != "constant":
        raise ValueError(f"device_transforms Pad needs size= with constant padding (no size_divisor / "
                         f"pad_to_square): {pd}")
    size = pd["size"]
    Wp, Hp = (int(size), int(size)) if isinstance(size, (int, float)) else (int(size[0]), int(size[1]))
    if Hp % pad_size_divisor or Wp % pad_size_divisor:
        raise ValueError(f"device_transforms Pad size {size} must be a multiple of pad_size_divisor {pad_size_divisor}")
    pv = pd.get("pad_val", 0)
    pv = pv.get("img", 0) if isinstance(pv, dict) else pv
    pv = tuple(float(v) for v in pv) if isinstance(pv, (tuple, list)) else (float(pv),) * 3
    if len(pv) != 3:
        raise ValueError(f"device_transforms Pad pad_val must be one value or three: {pd}")
    return scale, (Hp, Wp), pv


@MODELS.register_module(force=True)
class DetDataPreprocessor(BaseModule):
    def __init__(self, mean=None, std=None, pad_size_divisor: int = 1, pad_value: float = 0, pad_mask: bool = False,
                 mask_pad_value: int = 0, pad_seg: bool = False, seg_pad_value: int = 255, bgr_to_rgb: bool = False,
                 rgb_to_bgr: bool = False, boxtype2tensor: bool = True, non_blocking: bool = False,
                 batch_augments=None, device_transforms=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert not (bgr_to_rgb and rgb_to_bgr), "bgr_to_rgb and rgb_to_bgr cannot both be set"
        assert (mean is None) == (std is None), "mean and std come together"
        self.channel_conversion = bool(bgr_to_rgb or rgb_to_bgr)
        self.pad_size_divisor, self.pad_value = int(pad_size_divisor), float(pad_value)
        self.device_transforms = None
        if device_transforms:
            self.device_transforms = _parse_device_transforms(device_transforms, self.pad_size_divisor)
        self._enable_normalize = mean is not None
        self._mean3 = self._std3 = None
        if self._enable_normalize:
            assert len(mean) in (1, 3) and len(std) in (1, 3)
            self._mean3 = tuple(float(m) for m in (mean if len(mean) == 3 else list(mean) * 3))
            self._std3 = tuple(float(m) for m in (std if len(std) == 3 else list(std) * 3))
            self.register_buffer("mean", torch.tensor(mean, dtype=torch.float32).view(-1, 1, 1), persistent=False)
            self.register_buffer("std", torch.tensor(std, dtype=torch.float32).view(-1, 1, 1), persistent=False)
        self.register_buffer("_dev", torch.zeros(1), persistent=False)

    @property
    def device(self) -> torch.device:
        return self._dev.device

    def _one(self, img: torch.Tensor) -> torch.Tensor:
        x = img.to(self.device, non_blocking=True)
        if self.channel_conversion and x.shape[0] == 3:
            x = x[[2, 1, 0], ...]
        x = x.float()
        if self._enable_normalize:
            x = (x - self.mean) / self.std
        return x

    def _norm3(self):
        return (self._mean3 or (0.0, 0.0, 0.0), self._std3 or (1.0, 1.0, 1.0), self.channel_conversion)

    @torch.no_grad()
    def forward(self, data: dict, training: bool = False, fuse_patch_embed: bool = False) -> dict:
        if training:
            raise NotImplementedError("rsprompter_b200 implements the inference path only")
        inputs, samples = data["inputs"], data.get("data_samples")
        if self.device_transforms is not None:
            return self._resize_pad(inputs, samples)
        d = self.pad_size_divisor
        if isinstance(inputs, torch.Tensor):          # default_collate: already a batch [N, C, H, W]
            assert inputs.dim() == 4, "inputs must be NCHW or a list of CHW tensors"
            imgs = [inputs[i] for i in range(inputs.shape[0])]
        else:
            imgs = list(inputs)
            assert all(t.dim() == 3 for t in imgs), "inputs must be NCHW or a list of CHW tensors"
        pad_shapes = [(int(math.ceil(t.shape[1] / d)) * d, int(math.ceil(t.shape[2] / d)) * d) for t in imgs]
        H = int(math.ceil(max(t.shape[1] for t in imgs) / d)) * d
        W = int(math.ceil(max(t.shape[2] for t in imgs) / d)) * d
        u8 = self.device.type == "cuda" and all(t.dtype == torch.uint8 and t.shape[0] == 3 for t in imgs)
        if u8 and fuse_patch_embed and H % 16 == 0 and W % 16 == 0 and all(tuple(t.shape[1:]) == (H, W) for t in imgs):
            # the raw bytes are the batch: normalisation happens inside the patch-embed operand loader
            if isinstance(inputs, torch.Tensor) and (inputs.is_contiguous() or inputs.permute(0, 2, 3, 1).is_contiguous()):
                batch = inputs.to(self.device, non_blocking=True)
            else:
                batch = torch.stack([t.to(self.device, non_blocking=True) for t in imgs]).contiguous()
            batch.rsp_norm = self._norm3()
        elif u8:
            batch = torch.empty((len(imgs), 3, H, W), dtype=torch.float32, device=self.device)
            mean, std, swap = self._norm3()
            for i, t in enumerate(imgs):              # one kernel per image: flip + normalise + pad into its slot
                _lib.preprocess_u8(t.to(self.device, non_blocking=True), batch[i], mean, std, swap, self.pad_value)
        else:
            xs = [self._one(t) for t in imgs]
            batch = torch.full((len(xs), xs[0].shape[0], H, W), self.pad_value, dtype=torch.float32, device=self.device)
            for i, t in enumerate(xs):                # stack_batch: pad bottom / right
                batch[i, :, :t.shape[1], :t.shape[2]] = t
        if samples is None:
            samples = [DetDataSample(metainfo=dict(img_shape=tuple(t.shape[1:]), ori_shape=tuple(t.shape[1:]),
                                                   scale_factor=(1.0, 1.0))) for t in imgs]
        for ds, ps in zip(samples, pad_shapes):
            ds.set_metainfo(dict(batch_input_shape=(H, W), pad_shape=ps))
        return dict(inputs=batch, data_samples=samples)

    def _resize_pad(self, inputs, samples) -> dict:
        """device_transforms: uint8 CHW images of any sizes -> fp32 [B, 3, Hp, Wp] by one rsp_resize_pad_u8 launch,
        the metainfo of Resize + Pad written into the samples."""
        scale, (Hp, Wp), pad = self.device_transforms
        imgs = [inputs[i] for i in range(inputs.shape[0])] if isinstance(inputs, torch.Tensor) else list(inputs)
        for t in imgs:
            if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[0] != 3:
                raise ValueError("device_transforms take uint8 [3, h, w] images (LoadImageFromFile without "
                                 f"to_float32), got {getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))}")
        if self.device.type != "cuda":
            raise RuntimeError("device_transforms run on the GPU: move the preprocessor to a CUDA device")
        sizes = [rescale_size(t.shape[1:], scale) for t in imgs]
        for t, (nh, nw) in zip(imgs, sizes):
            if nh > Hp or nw > Wp:
                raise ValueError(f"a {tuple(t.shape[1:])} image resized by scale {scale} is {nh} x {nw}, larger than "
                                 f"the Pad size {Hp} x {Wp}")
        if all(t.is_cuda for t in imgs):
            dev = [t.to(self.device) for t in imgs]
        else:   # the original bytes of the whole batch in one pinned host -> device copy
            counts = [t.numel() for t in imgs]
            host = torch.empty(sum(counts), dtype=torch.uint8, pin_memory=True)
            offs = [0]
            for t, n in zip(imgs, counts):
                host[offs[-1]:offs[-1] + n].view(t.shape).copy_(t)
                offs.append(offs[-1] + n)
            flat = host.to(self.device, non_blocking=True)
            dev = [flat[o:o + n].view(t.shape) for t, o, n in zip(imgs, offs, counts)]
        batch = torch.empty((len(imgs), 3, Hp, Wp), dtype=torch.float32, device=self.device)
        mean, std, swap = self._norm3()
        _lib.resize_pad_u8(dev, sizes, batch, mean, std, swap, pad)
        if samples is None:
            samples = [DetDataSample(metainfo={}) for _ in imgs]
        for ds, t, s in zip(samples, imgs, sizes):
            meta = resize_metainfo(t.shape[1:], s, (Hp, Wp))
            if "ori_shape" in ds.metainfo:
                meta.pop("ori_shape")
            ds.set_metainfo(dict(meta, batch_input_shape=(Hp, Wp), pad_shape=(Hp, Wp)))
        return dict(inputs=batch, data_samples=samples)


__all__ = ["DetDataPreprocessor", "rescale_size", "resize_metainfo"]
