"""RSPrompter-anchor heads on the H100 kernels: RPNHead -> RSPrompterAnchorRoIPromptHead
(SingleRoIExtractor + Shared2FCBBoxHead) -> RSPrompterAnchorMaskHead -> SAM mask decoder.

Reference: mmdet/models/dense_heads/rpn_head.py:22-304, roi_heads/standard_roi_head.py:292-345,
roi_extractors/single_level_roi_extractor.py:55-119, bbox_heads/bbox_head.py:425-571,
layers/bbox_nms.py:13-105, mmdet/rsprompter/models.py:1366-1784 (M:).

The reference loops over images and levels in Python with data-dependent shapes (nonzero, boolean
indexing, per-image NMS calls -> dozens of host syncs per batch).  Here every stage is batched over
the B images with fixed-size padded candidate lists (score -1 = filtered / padding):
    level top-k (torch.topk on the logits; sigmoid is monotone) -> rsp_rpn_decode
    -> per-image score sort -> rsp_nms_batched (level offsets) -> rsp_compact_keep (<= 1000 proposals)
    -> rsp_roi_align_nhwc (7x7, extra sine PE sampled on the fly) -> FC GEMMs -> rsp_bbox_cls_decode
    -> sort -> rsp_nms_batched (class offsets) -> rsp_compact_keep (<= 100 detections)
    -> rsp_roi_align_nhwc (14x14) -> prompt GEMMs -> SAM decoder -> rsp_mask_paste
with a single device->host read of the per-image detection counts at the very end.
torch.topk / torch.sort are used as device-side index plumbing.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from . import _lib
from .necks import (_BN, _ConvT, _PrepMixin, _Slot, _conv, conv1x1, conv3x3, convT2x2, prep_conv, prep_convT,
                    to_nhwc_bf16)
from .registry import MODELS, BaseModule, ConfigDict, InstanceData
from .sam_encoder import _Affine


def _cfg(d) -> ConfigDict:
    return d if isinstance(d, ConfigDict) else ConfigDict(d or {})


# keys of an mmcv batched_nms config this package runs, per type; a key outside these raises instead of being ignored.
# offset, class_agnostic and split_thr are accepted at their mmcv defaults only.
_NMS_KEYS = {"nms": ("iou_threshold",), "soft_nms": ("iou_threshold", "sigma", "min_score", "method")}
_NMS_DEFAULTS = dict(offset=0, class_agnostic=False, split_thr=10000)


def parse_nms_cfg(nms) -> dict:
    """Validate a test_cfg ``nms`` dict (mmcv batched_nms nms_cfg) -> dict(type, iou_threshold[, sigma, min_score,
    method]) with mmcv's defaults filled in.  Raises ValueError naming an unsupported type, key or method."""
    d = dict(nms or {})
    typ = d.pop("type", "nms")
    if typ not in _NMS_KEYS:
        raise ValueError(f"nms type {typ!r} is not supported (supported: {', '.join(_NMS_KEYS)})")
    for k, v in _NMS_DEFAULTS.items():
        if k in d and d.pop(k) != v:
            raise ValueError(f"nms {k}={nms[k]!r} is not supported (only {v!r})")
    extra = sorted(set(d) - set(_NMS_KEYS[typ]))
    if extra:
        raise ValueError(f"nms key(s) {extra} not supported for type {typ!r}")
    out = dict(type=typ)
    if "iou_threshold" in d:
        out["iou_threshold"] = float(d["iou_threshold"])
    if typ == "soft_nms":
        method = d.get("method", "linear")
        if method not in _lib.SOFT_NMS_METHODS:
            raise ValueError(f"soft_nms method {method!r} is not supported (supported: "
                             f"{', '.join(_lib.SOFT_NMS_METHODS)})")
        out.update(iou_threshold=float(d.get("iou_threshold", 0.3)), sigma=float(d.get("sigma", 0.5)),
                   min_score=float(d.get("min_score", 1e-3)), method=method)
        if method == "gaussian" and not out["sigma"] > 0:
            raise ValueError(f"soft_nms sigma must be > 0 for method 'gaussian', got {out['sigma']}")
    return out


def _soft_nms_input_order(scores: torch.Tensor, boxes: torch.Tensor, ids: torch.Tensor, K: int, num_groups: int,
                          nms: dict):
    """Soft-NMS of each image's valid candidates (score >= 0) in their array order, which is mmcv's input order
    (ties and the serial loop's swaps depend on it): the valid ones are moved to the front, order kept, on the
    device.  -> boxes [B, K, 4], decayed scores [B, K], ids [B, K], counts int32 [B]."""
    invalid = (scores < 0).to(torch.uint8)
    _, order = torch.sort(invalid, dim=1, stable=True)
    s = torch.gather(scores, 1, order).contiguous()
    b = torch.gather(boxes, 1, order[:, :, None].expand(-1, -1, 4)).contiguous()
    i = torch.gather(ids, 1, order).contiguous()
    nvalid = (invalid == 0).sum(dim=1).to(torch.int32)
    ob, os_, ol, _, cnt = _lib.soft_nms_batched(b, s, i, nvalid, num_groups, nms["iou_threshold"], nms["sigma"],
                                                nms["min_score"], nms["method"], K=K)
    return ob, os_, ol, cnt


# ------------------------------------------------------------------------------ small registry types
@MODELS.register_module(force=True)
class AnchorGenerator:
    """mmdet AnchorGenerator (prior_generators/anchor_generator.py:14-301), scale-major, centre offset 0."""

    def __init__(self, strides, ratios, scales=None, base_sizes=None, scale_major=True,
                 octave_base_scale=None, scales_per_octave=None, centers=None, center_offset=0.0,
                 use_box_type=False):
        assert scales is not None and scale_major and centers is None and center_offset == 0.0
        self.strides = [s if isinstance(s, int) else s[0] for s in strides]
        self.base_sizes = list(base_sizes) if base_sizes is not None else list(self.strides)
        self.scales = torch.tensor(scales, dtype=torch.float32)
        self.ratios = torch.tensor(ratios, dtype=torch.float32)

    @property
    def num_base_priors(self):
        return [self.scales.numel() * self.ratios.numel()] * len(self.strides)

    def base_anchors(self, level: int) -> torch.Tensor:
        bs = float(self.base_sizes[level])
        hr = torch.sqrt(self.ratios)
        wr = 1 / hr
        ws = (bs * wr[:, None] * self.scales[None, :]).view(-1)
        hs = (bs * hr[:, None] * self.scales[None, :]).view(-1)
        return torch.stack([-0.5 * ws, -0.5 * hs, 0.5 * ws, 0.5 * hs], dim=-1)


@MODELS.register_module(force=True)
class DeltaXYWHBBoxCoder:
    def __init__(self, target_means=(0., 0., 0., 0.), target_stds=(1., 1., 1., 1.), clip_border=True,
                 add_ctr_clamp=False, ctr_clamp=32, use_box_type=False):
        assert all(m == 0 for m in target_means) and clip_border and not add_ctr_clamp
        self.means, self.stds = tuple(target_means), tuple(target_stds)
        self.encode_size = 4


@MODELS.register_module(force=True)
class RoIAlign:
    """Config holder for mmcv.ops.RoIAlign; the arithmetic is rsp_roi_align_nhwc."""

    def __init__(self, output_size, spatial_scale=1.0, sampling_ratio=0, pool_mode="avg", aligned=True,
                 use_torchvision=False):
        assert sampling_ratio == 0 and pool_mode == "avg" and aligned
        self.output_size = output_size if isinstance(output_size, int) else output_size[0]


@MODELS.register_module(force=True)
class SingleRoIExtractor(BaseModule):
    def __init__(self, roi_layer, out_channels, featmap_strides, finest_scale=56, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        layer = dict(roi_layer)
        assert layer.pop("type") == "RoIAlign"
        self.roi_layer = RoIAlign(**layer)
        self.out_channels = out_channels
        self.featmap_strides = list(featmap_strides)
        self.finest_scale = finest_scale
        self.num_inputs = len(featmap_strides)

    def extract(self, feats: list, rois: torch.Tensor, pes: list | None = None) -> torch.Tensor:
        """-> bf16 [n, P*P*C] in (ph, pw, c) order."""
        n = self.num_inputs
        return _lib.roi_align_nhwc(feats[:n], rois, self.roi_layer.output_size, self.featmap_strides,
                                   pes[:n] if pes is not None else None, float(self.finest_scale))


# ------------------------------------------------------------------------------ RPN
@MODELS.register_module(force=True)
class RPNHead(_PrepMixin, BaseModule):
    """rpn_head.py:22-304 (inference half)."""

    def __init__(self, in_channels, feat_channels=256, num_classes=1, anchor_generator=None, bbox_coder=None,
                 num_convs=1, loss_cls=None, loss_bbox=None, train_cfg=None, test_cfg=None, init_cfg=None,
                 **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert num_convs == 1 and num_classes == 1
        self.prior_generator = MODELS.build(anchor_generator)
        self.bbox_coder = MODELS.build(bbox_coder)
        self.test_cfg = _cfg(test_cfg)
        self._nms = parse_nms_cfg(self.test_cfg.get("nms"))
        A = self.prior_generator.num_base_priors[0]
        self.num_base_priors = A
        self.rpn_conv = _conv(feat_channels, in_channels, 3)
        self.rpn_cls = _conv(A, feat_channels, 1)
        self.rpn_reg = _conv(A * 4, feat_channels, 1)
        self._init_prep()

    @torch.no_grad()
    def _prepare(self):
        A = self.num_base_priors
        wc, bc = prep_conv(self.rpn_conv.weight, self.rpn_conv.bias)
        w = torch.cat([self.rpn_cls.weight, self.rpn_reg.weight], dim=0)
        b = torch.cat([self.rpn_cls.bias, self.rpn_reg.bias], dim=0)
        wh, bh = prep_conv(w, b, pad_out=((5 * A + 31) // 32) * 32)   # one GEMM for cls + reg
        dev = self.rpn_conv.weight.device
        anchors = [self.prior_generator.base_anchors(l).to(dev).contiguous()
                   for l in range(len(self.prior_generator.strides))]
        self._prep = dict(conv=(wc, bc), head=(wh, bh), anchors=anchors)
        return self._prep

    @torch.no_grad()
    def predict_nhwc(self, feats: list, img_hw: tuple, capture: dict | None = None,
                     img_shapes: torch.Tensor | None = None):
        """feats: bf16 NHWC levels -> proposals fp32 [B, K, 4], scores [B, K], counts int32 [B].
        img_shapes: device fp32 [B, 2] per-image (h, w) the boxes are clipped to (img_meta['img_shape'],
        rpn_head.py:208-215); None = the batch shape img_hw for every image.
        capture (tests): receives the raw per-level head outputs (and, with soft_nms, the NMS candidates)."""
        p = self._prep or self._prepare()
        cfg = self.test_cfg
        nms_pre, K = int(cfg.get("nms_pre", 1000)), int(cfg.get("max_per_img", 1000))
        A = self.num_base_priors
        B = feats[0].shape[0]
        dev = feats[0].device
        per_level = []
        for x in feats:
            H, W = x.shape[1], x.shape[2]
            per_level.append(min(nms_pre, H * W * A) if nms_pre > 0 else H * W * A)
        n = sum(per_level)
        boxes = torch.empty(B, n, 4, device=dev, dtype=torch.float32)
        scores = torch.empty(B, n, device=dev, dtype=torch.float32)
        ids = torch.empty(B, n, device=dev, dtype=torch.int64)
        off = 0
        for l, x in enumerate(feats):
            _, H, W, _ = x.shape
            y = conv3x3(x, *p["conv"], act="relu")
            out = _lib.gemm(y.reshape(B * H * W, -1), *p["head"], out_dtype=torch.float32)   # [B*H*W, 32]
            if capture is not None:
                capture.setdefault("head_out", []).append(out.view(B, H, W, -1))
            logits = out.view(B, H * W, -1)[:, :, :A].reshape(B, H * W * A)
            k = per_level[l]
            # rpn_head.py:206-212: descending sort, first nms_pre
            _, idx = torch.topk(logits, k, dim=1, largest=True, sorted=True)
            _lib.rpn_decode(out, idx.contiguous(), B, H, W, A, self.prior_generator.strides[l],
                            p["anchors"][l], img_hw, float(cfg.get("min_bbox_size", 0)), boxes, scores, off,
                            stds=self.bbox_coder.stds, img_shapes=img_shapes)
            ids[:, off:off + k] = l
            off += k
        if self._nms["type"] == "soft_nms":   # candidates in level order, each level's top-k in descending order
            if capture is not None:
                capture["candidates"] = (boxes, scores, ids)
            pb, ps, _, cnt = _soft_nms_input_order(scores, boxes, ids, K, len(feats), self._nms)
            return pb, ps, cnt
        # batched_nms sorts by score internally; filtered boxes (score -1) sink to the end
        s_sorted, order = torch.sort(scores, dim=1, descending=True, stable=True)
        b_sorted = torch.gather(boxes, 1, order[:, :, None].expand(-1, -1, 4)).contiguous()
        i_sorted = torch.gather(ids, 1, order).contiguous()
        nvalid = (s_sorted >= 0).sum(dim=1).to(torch.int32)
        keep = _lib.nms_batched(b_sorted, i_sorted, nvalid, float(cfg.nms.get("iou_threshold", 0.7)), max_keep=K)
        pb, ps, _, _, cnt = _lib.compact_keep(keep, b_sorted, s_sorted.contiguous(), None, K)
        return pb, ps, cnt

    def forward(self, x):
        """Reference signature: tuple of NCHW maps -> (cls_scores, bbox_preds) lists (rpn_head.py:80-97)."""
        p = self._prep or self._prepare()
        A = self.num_base_priors
        cls, reg = [], []
        for f in x:
            f = to_nhwc_bf16(f)
            B, H, W, _ = f.shape
            y = conv3x3(f, *p["conv"], act="relu")
            out = _lib.gemm(y.reshape(B * H * W, -1), *p["head"], out_dtype=torch.float32).view(B, H, W, -1)
            cls.append(out[..., :A].permute(0, 3, 1, 2).contiguous())
            reg.append(out[..., A:5 * A].permute(0, 3, 1, 2).contiguous())
        return cls, reg


# ------------------------------------------------------------------------------ bbox head
@MODELS.register_module(force=True)
class Shared2FCBBoxHead(_PrepMixin, BaseModule):
    """convfc_bbox_head.py Shared2FCBBoxHead: flatten -> 2 x (FC + ReLU) -> fc_cls / fc_reg."""

    def __init__(self, in_channels=256, fc_out_channels=1024, roi_feat_size=7, num_classes=80, bbox_coder=None,
                 reg_class_agnostic=False, loss_cls=None, loss_bbox=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert not reg_class_agnostic
        self.num_classes, self.roi_feat_size, self.in_channels = num_classes, roi_feat_size, in_channels
        self.bbox_coder = MODELS.build(bbox_coder)
        k = in_channels * roi_feat_size * roi_feat_size
        self.shared_fcs = nn.ModuleList([_Affine((fc_out_channels, k)), _Affine((fc_out_channels, fc_out_channels))])
        self.fc_cls = _Affine((num_classes + 1, fc_out_channels))
        self.fc_reg = _Affine((4 * num_classes, fc_out_channels))
        self._init_prep()

    @torch.no_grad()
    def _prepare(self):
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()  # noqa: E731
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        C, P = self.in_channels, self.roi_feat_size
        # reference flattens (C, P, P); our RoIAlign writes (P, P, C): permute the FC columns once
        w0 = self.shared_fcs[0].weight.view(-1, C, P, P).permute(0, 2, 3, 1).reshape(-1, C * P * P)
        nc = self.num_classes
        wh = torch.cat([self.fc_cls.weight, self.fc_reg.weight], dim=0)
        bh = torch.cat([self.fc_cls.bias, self.fc_reg.bias], dim=0)
        pad = ((wh.shape[0] + 31) // 32) * 32 - wh.shape[0]
        wh = torch.cat([wh, wh.new_zeros(pad, wh.shape[1])])
        bh = torch.cat([bh, bh.new_zeros(pad)])
        self._prep = dict(fc0=(bf(w0), f32(self.shared_fcs[0].bias)),
                          fc1=(bf(self.shared_fcs[1].weight), f32(self.shared_fcs[1].bias)),
                          head=(bf(wh), f32(bh)), ncls=nc + 1, nreg=4 * nc)
        return self._prep

    @torch.no_grad()
    def forward_rows(self, roi_feats: torch.Tensor):
        """roi_feats bf16 [n, P*P*C] -> (cls fp32 [n, C+1], reg fp32 [n, 4C]) as views of one GEMM output."""
        p = self._prep or self._prepare()
        x = _lib.gemm(roi_feats, *p["fc0"], act="relu")
        x = _lib.gemm(x, *p["fc1"], act="relu")
        out = _lib.gemm(x, *p["head"], out_dtype=torch.float32)
        return out[:, :p["ncls"]], out[:, p["ncls"]:p["ncls"] + p["nreg"]]


# ------------------------------------------------------------------------------ mask head
@MODELS.register_module(force=True)
class RSPrompterAnchorMaskHead(_PrepMixin, BaseModule):
    """M:1596-1784 (inference half): RoI features -> 5 point embeddings -> SAM decoder."""

    def __init__(self, mask_decoder, in_channels, roi_feat_size=14, per_pointset_point=5, with_sincos=True,
                 multimask_output=False, attention_similarity=None, target_embedding=None,
                 output_attentions=None, class_agnostic=False, loss_mask=None, init_cfg=None, *args, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        self.in_channels, self.roi_feat_size = in_channels, roi_feat_size
        self.per_pointset_point, self.with_sincos = per_pointset_point, with_sincos
        self.multimask_output, self.class_agnostic = multimask_output, class_agnostic
        self.mask_decoder = MODELS.build(mask_decoder)
        pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name=mask_decoder.get("hf_pretrain_name"),
                               init_cfg=mask_decoder.get("init_cfg")))
        self.no_mask_embed = pe.prompt_encoder.no_mask_embed
        ns = 2 if with_sincos else 1
        c = in_channels
        self.point_emb = nn.Sequential(
            _conv(c, c, 3), _BN(c), _Slot(), _Slot(), _Affine((c, c * roi_feat_size ** 2 // 4)), _Slot(),
            _Affine((c, c)), _Slot(), _Affine((c * ns * per_pointset_point, c)))
        self._init_prep()

    def init_weights(self):
        pass

    @torch.no_grad()
    def _prepare(self):
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()  # noqa: E731
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        pe = self.point_emb
        C, P = self.in_channels, self.roi_feat_size // 2
        w4 = pe[4].weight.view(-1, C, P, P).permute(0, 2, 3, 1).reshape(-1, C * P * P)   # (C,P,P) -> (P,P,C)
        self._prep = dict(conv=prep_conv(pe[0].weight, pe[0].bias, pe[1]), fc4=(bf(w4), f32(pe[4].bias)),
                          fc6=(bf(pe[6].weight), f32(pe[6].bias)), fc8=(bf(pe[8].weight), f32(pe[8].bias)),
                          no_mask=f32(self.no_mask_embed.weight.reshape(-1)))
        return self._prep

    @torch.no_grad()
    def prompts_from_roi_feats(self, roi_feats: torch.Tensor) -> torch.Tensor:
        """roi_feats bf16 [N, 14*14*C] (ph, pw, c) -> sparse embeddings fp32 [N, P, C] (M:1669-1672)."""
        p = self._prep or self._prepare()
        N = roi_feats.shape[0]
        R, C = self.roi_feat_size, self.in_channels
        x = conv3x3(roi_feats.view(N, R, R, C), *p["conv"], act="relu", stride=2)      # [N, 7, 7, C]
        x = _lib.gemm(x.reshape(N, -1), *p["fc4"], act="relu")
        x = _lib.gemm(x, *p["fc6"], act="relu")
        x = _lib.gemm(x, *p["fc8"], out_dtype=torch.float32)                           # [N, P * ns * C]
        x = x.view(N, self.per_pointset_point, -1)
        return _lib.sin_fold(x.contiguous()) if self.with_sincos else x

    @torch.no_grad()
    def decode(self, roi_feats: torch.Tensor, emb_rows: torch.Tensor, pos_rows: torch.Tensor, hw: tuple,
               prompt_img: torch.Tensor):
        """-> low-res mask logits fp32 [N, n_out, 4h, 4w], iou [N, n_out] (M:1659-1698)."""
        p = self._prep or self._prepare()
        sparse = self.prompts_from_roi_feats(roi_feats)
        return self.mask_decoder.mask_decoder.decode(emb_rows, pos_rows, sparse, hw, prompt_img=prompt_img,
                                                     dense_vec=p["no_mask"],
                                                     multimask_output=self.multimask_output)


# ------------------------------------------------------------------------------ RoI head
def _predict_bboxes(head, feats: list, proposals: torch.Tensor, prop_counts: torch.Tensor, img_hw: tuple,
                    pes: list | None = None, capture: dict | None = None, img_shapes: torch.Tensor | None = None):
    """StandardRoIHead.predict_bbox (standard_roi_head.py:292-345) + BBoxHead._predict_by_feat_single
    (bbox_head.py:505-571) + multiclass_nms (bbox_nms.py:13-105), batched over the B images.
    -> detections bboxes fp32 [B, M, 4], scores [B, M], labels int64 [B, M], counts int32 [B].
    nms type 'soft_nms': the scores are the decayed ones and the rows are in selection order."""
    cfg = head.test_cfg
    B, K, _ = proposals.shape
    dev = proposals.device
    bidx = torch.arange(B, device=dev, dtype=torch.float32).view(B, 1, 1).expand(B, K, 1)
    rois = torch.cat([bidx, proposals], dim=2).reshape(B * K, 5).contiguous()
    valid = (torch.arange(K, device=dev).view(1, K) < prop_counts.view(B, 1)).reshape(-1).to(torch.uint8)
    feats7 = head.bbox_roi_extractor.extract(feats, rois, pes)
    cls, reg = head.bbox_head.forward_rows(feats7)
    if capture is not None:
        capture.update(roi_feats7=feats7, cls=cls, reg=reg, rois=rois)
    C = head.bbox_head.num_classes
    s, b, lab = _lib.bbox_cls_decode(cls, reg, rois, valid.contiguous(), C, img_hw, float(cfg.get("score_thr", 0.05)),
                                     stds=head.bbox_head.bbox_coder.stds, img_shapes=img_shapes)
    n = K * C
    s, b, lab = s.view(B, n), b.view(B, n, 4), lab.view(B, n)
    if head._nms["type"] == "soft_nms":   # candidates (RoI, class) with score > score_thr, RoI-major
        if capture is not None:
            capture["candidates"] = (b, s, lab)
        return _soft_nms_input_order(s, b, lab, int(cfg.get("max_per_img", 100)), C, head._nms)
    s_sorted, order = torch.sort(s, dim=1, descending=True, stable=True)
    b_sorted = torch.gather(b, 1, order[:, :, None].expand(-1, -1, 4)).contiguous()
    l_sorted = torch.gather(lab, 1, order).contiguous()
    nvalid = (s_sorted >= 0).sum(dim=1).to(torch.int32)
    M = int(cfg.get("max_per_img", 100))
    keep = _lib.nms_batched(b_sorted, l_sorted, nvalid, float(cfg.nms.get("iou_threshold", 0.5)), max_keep=M)
    db, ds, dl, _, cnt = _lib.compact_keep(keep, b_sorted, s_sorted.contiguous(), l_sorted, M)
    return db, ds, dl, cnt


def _detection_rois(db: torch.Tensor) -> torch.Tensor:
    B, M, _ = db.shape
    bidx = torch.arange(B, device=db.device, dtype=torch.float32).view(B, 1, 1).expand(B, M, 1)
    return torch.cat([bidx, db], dim=2).reshape(B * M, 5).contiguous()


def sine_pe_rows(h: int, w: int, num_feats: int, device, temperature: int = 10000,
                 scale: float = 2 * math.pi, eps: float = 1e-6) -> torch.Tensor:
    """SinePositionalEncoding(normalize=True) on an all-valid h x w mask -> fp32 [1, 2F, h, w]
    (positional_encoding.py:60-110).  A constant per size: evaluated once at set-up."""
    y = torch.arange(1, h + 1, dtype=torch.float32, device=device).view(1, h, 1).repeat(1, 1, w)
    x = torch.arange(1, w + 1, dtype=torch.float32, device=device).view(1, 1, w).repeat(1, h, 1)
    y = y / (y[:, -1:, :] + eps) * scale
    x = x / (x[:, :, -1:] + eps) * scale
    dim_t = torch.arange(num_feats, dtype=torch.float32, device=device)
    dim_t = temperature ** (2 * (dim_t // 2) / num_feats)
    px, py = x[:, :, :, None] / dim_t, y[:, :, :, None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=4).view(1, h, w, -1)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=4).view(1, h, w, -1)
    return torch.cat((py, px), dim=3).permute(0, 3, 1, 2)


@MODELS.register_module(force=True)
class RSPrompterAnchorRoIPromptHead(BaseModule):
    """M:1366-1593 (inference half) over StandardRoIHead.predict_bbox (standard_roi_head.py:292-345)."""

    def __init__(self, with_extra_pe=False, bbox_roi_extractor=None, bbox_head=None, mask_roi_extractor=None,
                 mask_head=None, shared_head=None, train_cfg=None, test_cfg=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert shared_head is None
        self.bbox_roi_extractor = MODELS.build(bbox_roi_extractor)
        self.bbox_head = MODELS.build(bbox_head)
        self.mask_roi_extractor = MODELS.build(mask_roi_extractor)
        self.mask_head = MODELS.build(mask_head)
        self.test_cfg = _cfg(test_cfg)
        self._nms = parse_nms_cfg(self.test_cfg.get("nms"))
        self.with_extra_pe = with_extra_pe
        self._pe_cache: dict = {}

    def init_weights(self):
        pass

    def _extra_pe(self, feats: list) -> list | None:
        """Per-level fp32 [H, W, C] tables of the bilinearly resized sine PE (M:1566-1574)."""
        if not self.with_extra_pe:
            return None
        key = tuple((f.shape[1], f.shape[2]) for f in feats) + (str(feats[0].device),)
        if key not in self._pe_cache:
            h, w, c = feats[0].shape[1], feats[0].shape[2], feats[0].shape[3]
            pe = sine_pe_rows(h, w, c // 2, feats[0].device)
            tabs = []
            for f in feats:
                t = torch.nn.functional.interpolate(pe, size=(f.shape[1], f.shape[2]), mode="bilinear",
                                                    align_corners=False)
                tabs.append(t[0].permute(1, 2, 0).contiguous())
            self._pe_cache = {key: tabs}
        return self._pe_cache[key]

    @torch.no_grad()
    def predict_nhwc(self, feats: list, proposals: torch.Tensor, prop_counts: torch.Tensor, img_hw: tuple,
                     emb_rows: torch.Tensor, pos_rows: torch.Tensor, emb_hw: tuple, capture: dict | None = None,
                     img_shapes: torch.Tensor | None = None):
        """proposals fp32 [B, K, 4] (zero padded), prop_counts int32 [B].
        -> dict(bboxes [B, M, 4], scores [B, M], labels [B, M], counts int32 [B], mask_logits [B*M, 1, 4h, 4w])."""
        B, dev = proposals.shape[0], proposals.device
        pes = self._extra_pe(feats)
        if pes is not None:       # x = [xi + pe_i] once per level (M:1566-1574); both extractors then read bf16 only
            n_lvl = max(self.bbox_roi_extractor.num_inputs, self.mask_roi_extractor.num_inputs)
            feats = [_lib.add_table_bf16(f, t) for f, t in zip(feats[:n_lvl], pes[:n_lvl])] + list(feats[n_lvl:])
            pes = None
        db, ds, dl, cnt = _predict_bboxes(self, feats, proposals, prop_counts, img_hw, pes, capture, img_shapes)
        M = db.shape[1]
        # mask branch (M:1511-1550): RoIs = detections
        mrois = _detection_rois(db)
        feats14 = self.mask_roi_extractor.extract(feats, mrois, pes)
        if capture is not None:
            capture.update(roi_feats14=feats14, mask_rois=mrois)
        prompt_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(M).contiguous()
        logits, iou = self.mask_head.decode(feats14, emb_rows, pos_rows, emb_hw, prompt_img)
        return dict(bboxes=db, scores=ds, labels=dl, counts=cnt, mask_logits=logits, iou=iou)


# ------------------------------------------------------------------------------ stock Mask R-CNN heads (SAMSegMaskRCNN)
class _ConvOnly(nn.Module):
    """mmcv ConvModule(norm_cfg=None): conv (+ ReLU); parameters live under ``.conv``."""

    def __init__(self, cin: int, cout: int, k: int = 3):
        super().__init__()
        self.conv = _conv(cout, cin, k)


@MODELS.register_module(force=True)
class FCNMaskHead(_PrepMixin, BaseModule):
    """mmdet/models/roi_heads/mask_heads/fcn_mask_head.py (inference half): num_convs x (conv3x3 + ReLU) ->
    ConvTranspose2d(k2, s2) + ReLU -> 1x1 conv_logits (:31-126 build, :128-147 forward); the per-class channel is picked
    by the detection label (:377-379)."""

    def __init__(self, num_convs=4, roi_feat_size=14, in_channels=256, conv_kernel_size=3, conv_out_channels=256,
                 num_classes=80, class_agnostic=False, upsample_cfg=None, conv_cfg=None, norm_cfg=None,
                 predictor_cfg=None, loss_mask=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        up = dict(upsample_cfg or dict(type="deconv", scale_factor=2))
        assert up.get("type") == "deconv" and up.get("scale_factor", 2) == 2 and conv_kernel_size == 3 and norm_cfg is None, \
            "FCNMaskHead is built as the RSPrompter configs use it (deconv x2, 3x3 convs, no norm)"
        self.num_convs, self.roi_feat_size, self.in_channels = num_convs, roi_feat_size, in_channels
        self.conv_out_channels, self.num_classes, self.class_agnostic = conv_out_channels, num_classes, class_agnostic
        self.convs = nn.ModuleList(
            _ConvOnly(in_channels if i == 0 else conv_out_channels, conv_out_channels) for i in range(num_convs))
        c_up = conv_out_channels if num_convs > 0 else in_channels
        self.upsample = _ConvT(c_up, conv_out_channels)
        self.conv_logits = _conv(1 if class_agnostic else num_classes, conv_out_channels, 1)
        self._init_prep()

    def init_weights(self):
        pass

    @torch.no_grad()
    def _prepare(self):
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        wl = self.conv_logits.weight.detach().reshape(self.conv_logits.weight.shape[0], -1)
        pad = ((wl.shape[0] + 31) // 32) * 32 - wl.shape[0]
        wl = torch.cat([wl, wl.new_zeros(pad, wl.shape[1])]).to(torch.bfloat16).contiguous()
        bl = torch.cat([f32(self.conv_logits.bias), self.conv_logits.bias.new_zeros(pad).float()])
        self._prep = dict(convs=[prep_conv(c.conv.weight, c.conv.bias) for c in self.convs],
                          up=prep_convT(self.upsample.weight, self.upsample.bias), logits=(wl, bl))
        return self._prep

    @torch.no_grad()
    def forward_rows(self, roi_feats: torch.Tensor) -> torch.Tensor:
        """roi_feats bf16 [N, R*R*C] in (ph, pw, c) order -> mask logits fp32 [N, 2R, 2R, n_cls (padded to 32)]."""
        p = self._prep or self._prepare()
        N, R, C = roi_feats.shape[0], self.roi_feat_size, self.in_channels
        x = roi_feats.view(N, R, R, C)
        if self.num_convs > 0 and C == self.conv_out_channels and _lib.conv3x3_ok(N, R + 2, R + 2, C):
            # RoI maps embedded in (R+2)^2 canvases: 128-pixel GEMM tiles are boxes of a 16x16 map, so the convolutions run
            # as implicit GEMMs (no im2col matrix: 2.6 GB of DRAM traffic per batch of 800 RoIs); the canvas border is the
            # convolutions' zero padding, restored after every layer.  The 2x deconv / 1x1 logits are per-pixel, so the
            # border only produces values that the final crop discards.
            S = R + 2
            canvas = torch.zeros(N, S, S, C, device=x.device, dtype=torch.bfloat16)
            canvas[:, 1:R + 1, 1:R + 1] = x
            x = canvas
            for i, (w, b) in enumerate(p["convs"]):
                x = conv3x3(x, w, b, act="relu")
                if i + 1 < len(p["convs"]):
                    _lib.zero_border_nhwc(x)
            x = convT2x2(x, *p["up"], act="relu")
            y = _lib.gemm(x.reshape(N * 4 * S * S, -1), *p["logits"], out_dtype=torch.float32).view(N, 2 * S, 2 * S, -1)
            return y[:, 2:2 * R + 2, 2:2 * R + 2]
        for w, b in p["convs"]:
            x = conv3x3(x, w, b, act="relu")
        x = convT2x2(x, *p["up"], act="relu")
        y = _lib.gemm(x.reshape(N * 4 * R * R, -1), *p["logits"], out_dtype=torch.float32)
        return y.view(N, 2 * R, 2 * R, -1)

    @torch.no_grad()
    def select(self, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """logits fp32 [N, h, w, C_pad], labels int64 [N] -> the label's channel fp32 [N, h, w] (:377-379)."""
        N, h, w, _ = logits.shape
        if self.class_agnostic:
            return logits[..., 0].contiguous()
        idx = labels.clamp(0, self.num_classes - 1).view(N, 1, 1, 1).expand(N, h, w, 1)
        return torch.gather(logits, 3, idx)[..., 0].contiguous()


@MODELS.register_module(force=True)
class StandardRoIHead(BaseModule):
    """mmdet/models/roi_heads/standard_roi_head.py (inference half): predict_bbox :292-345, predict_mask :347-419."""

    def __init__(self, bbox_roi_extractor=None, bbox_head=None, mask_roi_extractor=None, mask_head=None,
                 shared_head=None, train_cfg=None, test_cfg=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert shared_head is None
        self.bbox_roi_extractor = MODELS.build(bbox_roi_extractor)
        self.bbox_head = MODELS.build(bbox_head)
        self.with_mask = mask_head is not None
        if self.with_mask:
            self.mask_roi_extractor = MODELS.build(mask_roi_extractor) if mask_roi_extractor is not None else None
            self.mask_head = MODELS.build(mask_head)
        self.test_cfg = _cfg(test_cfg)
        self._nms = parse_nms_cfg(self.test_cfg.get("nms"))

    def init_weights(self):
        pass

    @torch.no_grad()
    def predict_nhwc(self, feats: list, proposals: torch.Tensor, prop_counts: torch.Tensor, img_hw: tuple,
                     capture: dict | None = None, img_shapes: torch.Tensor | None = None):
        """-> dict(bboxes [B, M, 4], scores [B, M], labels [B, M], counts int32 [B],
        mask_probs fp32 [B*M, 2R, 2R] = sigmoid of the label's mask channel (fcn_mask_head.py:358 / :377-379))."""
        db, ds, dl, cnt = _predict_bboxes(self, feats, proposals, prop_counts, img_hw, None, capture, img_shapes)
        out = dict(bboxes=db, scores=ds, labels=dl, counts=cnt)
        if self.with_mask:
            mrois = _detection_rois(db)
            ext = self.mask_roi_extractor or self.bbox_roi_extractor     # share_roi_extractor (:56-63)
            feats14 = ext.extract(feats, mrois, None)
            logits = self.mask_head.forward_rows(feats14)
            if capture is not None:
                capture.update(roi_feats14=feats14, mask_rois=mrois, mask_logits_all=logits)
            out["mask_probs"] = _lib.sigmoid_f32(self.mask_head.select(logits, dl.reshape(-1)))
        return out


__all__ = ["parse_nms_cfg", "FCNMaskHead", "StandardRoIHead", "AnchorGenerator", "DeltaXYWHBBoxCoder", "RoIAlign", "SingleRoIExtractor", "RPNHead",
           "Shared2FCBBoxHead", "RSPrompterAnchorMaskHead", "RSPrompterAnchorRoIPromptHead", "sine_pe_rows"]
