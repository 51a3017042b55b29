"""RSPrompterAnchor / RSPrompterQuery detectors (M:53-272): orchestration of the H100 modules.

``predict(batch_inputs, batch_data_samples, rescale=True)`` keeps the reference contract
(mmdet BaseDetector.forward mode='predict', detectors/base.py:58-99): it returns the data samples
with ``pred_instances`` holding ``bboxes``, ``scores``, ``labels`` and boolean ``masks`` (COCO RLE dicts with
``test_cfg.rle_masks``).  The query detectors follow ``test_cfg``'s ``instance_on`` / ``panoptic_on`` flags as the
reference does: ``panoptic_on`` (default True) adds ``pred_panoptic_seg`` (a ``PixelData`` with an int32 ``sem_seg``
[1, H, W]); ``pred_instances`` is set only with ``instance_on``.
Everything between the input tensor and the final per-image split runs on the device without
host synchronisation; the one device->host read is the per-image detection count.
"""
from __future__ import annotations

import torch

from . import _lib
from .necks import PseudoFeatureAggregator
from .registry import MODELS, BaseModule, ConfigDict, DetDataSample, InstanceData, PixelData, make_data_samples
from .results import ResultRecord, encode_mask_results
from .sam_encoder import MMPretrainSamVisionEncoder, SamVisionEncoderOutput


def _cfg(d) -> ConfigDict:
    return d if isinstance(d, ConfigDict) else ConfigDict(d or {})


class _SamDetectorBase(BaseModule):
    # ---- CUDA-graph replay of the device-resident forward ----------------------------------------------------
    # predict_raw() is ~420 launches with static shapes and no host synchronisation, so one captured graph per
    # input shape replays it without per-launch host work or inter-kernel launch gaps.  Opt-in
    # (enable_cuda_graphs()): capture allocates a private memory pool per shape.
    def enable_cuda_graphs(self, enabled: bool = True):
        """Replay the device-resident forward as one CUDA graph per input shape.  The graph's output buffers are
        reused by the next call with the same shape: predict() / predict_records() copy what they hand back, callers
        of _raw() must consume the result before calling again."""
        self._graphs = {} if enabled else None
        return self

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        if getattr(self, "_graphs", None):
            self._graphs = {}          # captured graphs hold the previous prepared weights: recapture on next use
        return out

    def _apply(self, fn, *args, **kwargs):
        if getattr(self, "_graphs", None):
            self._graphs = {}          # .to() / .cuda() / .half() move the parameters the graphs point at
        return super()._apply(fn, *args, **kwargs)

    def _raw(self, batch_inputs: torch.Tensor) -> dict:
        graphs = getattr(self, "_graphs", None)
        if graphs is None:
            return self.predict_raw(batch_inputs)
        shapes = getattr(batch_inputs, "rsp_img_shapes", None)
        key = (tuple(batch_inputs.shape), batch_inputs.dtype, tuple(batch_inputs.stride()),
               getattr(batch_inputs, "rsp_norm", None), shapes is not None)
        if key not in graphs:
            static_in = batch_inputs.to(next(self.parameters()).device, copy=True)   # also accepts a pinned host batch
            if hasattr(batch_inputs, "rsp_norm"):      # uint8 batch: normalisation rides along (DetDataPreprocessor)
                static_in.rsp_norm = batch_inputs.rsp_norm
            if shapes is not None:                     # per-image clip shapes: a static buffer refreshed per call
                static_in.rsp_img_shapes = shapes.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):          # warm-up: one-time attribute calls, caches, constant tables
                for _ in range(2):
                    self.predict_raw(static_in)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count
            with torch.cuda.graph(g):
                out = self.predict_raw(static_in)
            graphs[key] = (g, static_in, out, _lib.launch_count - n0)
        g, static_in, out, n_launch = graphs[key]
        static_in.copy_(batch_inputs, non_blocking=True)
        if shapes is not None:
            static_in.rsp_img_shapes.copy_(shapes, non_blocking=True)
        g.replay()
        _lib.launch_count += n_launch      # the replay launches the library's kernels again
        return out      # static output buffers: valid until the next call with this shape

    def _encode(self, batch_inputs: torch.Tensor):
        """-> (emb_rows fp32 [B*g*g, C], pos_rows fp32 [g*g, C], (g, g), emb_nhwc_bf16 | None, hidden | None)."""
        enc = self.backbone.vision_encoder
        want_hidden = not isinstance(self.backbone, MMPretrainSamVisionEncoder)
        # hidden states the aggregator reads leave the encoder as bf16 side outputs of the next layer's LN1
        sel = getattr(getattr(self.neck, "feature_aggregator", None), "select_layers", None)
        copies = {int(i): None for i in sel if int(i) < enc.arch.num_layers} if (want_hidden and sel is not None) else None
        emb, hidden, emb_nhwc = enc.encode(batch_inputs, want_hidden=want_hidden, bf16_copies=copies)
        if copies:
            hidden = tuple(copies.get(i, h) if copies.get(i) is not None else h for i, h in enumerate(hidden))
        B, g = emb_nhwc.shape[0], emb_nhwc.shape[1]
        sie = getattr(self, "shared_image_embedding", None)        # SAMSegMaskRCNN has no SAM decoder, hence no PE
        pos_rows = sie.shared_image_embedding.image_wide_rows(g) if sie is not None else None
        return emb_nhwc.reshape(B * g * g, -1), pos_rows, (g, g), emb_nhwc, hidden

    def extract_feat(self, batch_inputs: torch.Tensor):
        """Reference return convention (M:97-114): (x NCHW tuple, image_embeddings, image_positional_embeddings)."""
        vision_outputs = self.backbone(batch_inputs)
        if isinstance(vision_outputs, SamVisionEncoderOutput):
            image_embeddings, hidden = vision_outputs[0], vision_outputs[1]
        elif isinstance(vision_outputs, tuple):
            image_embeddings, hidden = vision_outputs[0], vision_outputs
        else:
            raise NotImplementedError
        size = image_embeddings.shape[-1]
        pe = self.shared_image_embedding.shared_image_embedding.image_wide_rows(size)
        pe = pe.view(size, size, -1).permute(2, 0, 1).unsqueeze(0).repeat(image_embeddings.shape[0], 1, 1, 1)
        x = self.neck(hidden)
        return x, image_embeddings, pe

    def _preprocess(self, data: dict) -> dict:
        """BaseModel.test_step's data_preprocessor(data, False); the detector lets its own preprocessor hand over the
        uint8 batch when the normalisation can be fused into the patch-embed operand loader."""
        if self.data_preprocessor is None:
            return data
        return self.data_preprocessor(data, False, fuse_patch_embed=True)

    def _new_record(self, B: int, M: int, hw: tuple, device) -> ResultRecord:
        """With CUDA graphs on, records alternate between two buffers per shape so that the previous step's record can
        still be in flight (side-stream gather / D2H) while this step writes the next one."""
        if getattr(self, "_graphs", None) is None:
            return ResultRecord(B, M, hw, device=device)
        pool = self.__dict__.setdefault("_rec_pool", {})
        key = (B, M, tuple(hw), str(device))
        slot = pool.setdefault(key, dict(i=0, recs=[ResultRecord(B, M, hw, device=device) for _ in range(2)]))
        slot["i"] ^= 1
        return slot["recs"][slot["i"]]

    @staticmethod
    def _attach_img_shapes(batch_data_samples, batch_inputs):
        """img_meta['img_shape'] of every image as a device fp32 [B, 2] tensor riding on the batch tensor
        (``rsp_img_shapes``) when any image is smaller than the batch shape (DetDataPreprocessor padding): the RPN and
        bbox-head decoders clip to it per image (rpn_head.py:208-215, bbox_head.py:545-548).  Nothing is attached when
        every img_shape equals the batch shape (the shipped Resize + Pad pipelines)."""
        hw = tuple(int(v) for v in batch_inputs.shape[-2:])
        shapes = [tuple(int(v) for v in tuple(ds.metainfo.get("img_shape", hw))[:2]) for ds in batch_data_samples]
        if all(s == hw for s in shapes):
            if hasattr(batch_inputs, "rsp_img_shapes"):      # the same tensor object went through a padded batch before
                del batch_inputs.rsp_img_shapes
            return batch_inputs
        t = torch.tensor(shapes, dtype=torch.float32).to(batch_inputs.device, non_blocking=True)
        batch_inputs.rsp_img_shapes = t
        return batch_inputs

    @staticmethod
    def _metas(batch_data_samples, batch_inputs):
        """-> (batch hw, per-image list of None (ori_shape == img_shape == batch shape, scale_factor 1: the fast
        batched post-process applies) or dict(ori_hw, crop_hw, scale_factor) for resized / padded images)."""
        hw = tuple(int(v) for v in batch_inputs.shape[-2:])
        out = []
        for ds in batch_data_samples:
            m = ds.metainfo
            sf = tuple(float(s) for s in m.get("scale_factor", (1.0, 1.0)))
            ori = tuple(int(v) for v in tuple(m.get("ori_shape", hw))[:2])
            if ori == hw and sf == (1.0, 1.0):
                out.append(None)
                continue
            # crop of the batch-sized map that holds the resized, unpadded image (M:1771-1773, M:681-685)
            crop = (min(int(ori[0] * sf[1]), hw[0]), min(int(ori[1] * sf[0]), hw[1]))
            out.append(dict(ori_hw=ori, crop_hw=crop, scale_factor=sf))
        return hw, out

    def _record_metas(self, batch_data_samples, batch_inputs, record):
        """predict_records with data samples -> (batch_inputs, metas, record hw).  metas is None when every image is at
        the batch shape with scale 1 (the batch-shape record path); otherwise the per-image _metas of resized images
        that all share one ori_shape, whose masks the record holds at its slots' top-left: record.hw must cover
        ori_shape (a new record is ori_shape with the width rounded up to 16, the bit kernels' store width)."""
        if batch_data_samples is None:
            return batch_inputs, None, None
        hw, metas = self._metas(batch_data_samples, batch_inputs)
        batch_inputs = self._attach_img_shapes(batch_data_samples, batch_inputs)
        if all(m is None for m in metas):
            return batch_inputs, None, None
        oris = {hw if m is None else m["ori_hw"] for m in metas}
        if len(oris) != 1:
            raise ValueError(f"predict_records writes one record shape: every image must share one ori_shape, got "
                             f"{sorted(oris)}")
        metas = [m or dict(ori_hw=hw, crop_hw=hw, scale_factor=(1.0, 1.0)) for m in metas]
        ori = metas[0]["ori_hw"]
        rhw = tuple(record.hw) if record is not None else (ori[0], (ori[1] + 15) // 16 * 16)
        if ori[0] > rhw[0] or ori[1] > rhw[1] or rhw[1] % 16:
            raise ValueError(f"a record of {rhw} cannot hold masks of ori_shape {ori} (needs H, W >= ori_shape and "
                             f"W % 16 == 0)")
        return batch_inputs, metas, rhw

    @staticmethod
    def _rescaled_boxes(boxes: torch.Tensor, metas: list) -> torch.Tensor:
        """boxes [B, M, 4] / scale_factor per image, the fp32 division predict(rescale=True) does."""
        sf = torch.tensor([list(m["scale_factor"]) * 2 for m in metas], dtype=torch.float32)
        return boxes / sf.to(boxes.device, non_blocking=True)[:, None, :]

    @staticmethod
    def _rle_masks(test_cfg, batch_data_samples):
        """With test_cfg.rle_masks, every pred_instances.masks becomes a list of COCO RLE dicts ({'size': [h, w],
        'counts': bytes}, h, w = the mask's size) encoded on the device in one batched call.  CocoMetric.process passes
        non-tensor masks through (coco_metric.py:364-367), so evaluation copies no mask pixel to the host."""
        if test_cfg is None or not test_cfg.get("rle_masks", False):
            return batch_data_samples
        insts = [ds.pred_instances for ds in batch_data_samples if "pred_instances" in ds]
        if not insts:           # panoptic-only results
            return batch_data_samples
        for inst, rles in zip(insts, encode_mask_results([inst.masks for inst in insts])):
            inst.masks = rles
        return batch_data_samples


@MODELS.register_module(force=True)
class RSPrompterAnchor(_SamDetectorBase):
    """M:53-170 over mmdet MaskRCNN / TwoStageDetector (detectors/two_stage.py:15-107)."""

    def __init__(self, shared_image_embedding, decoder_freeze=True, backbone=None, neck=None, rpn_head=None,
                 roi_head=None, train_cfg=None, test_cfg=None, data_preprocessor=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        test_cfg = _cfg(test_cfg)
        self.backbone = MODELS.build(backbone)
        self.neck = MODELS.build(neck)
        rpn = dict(rpn_head)
        rpn.update(train_cfg=None, test_cfg=test_cfg.get("rpn"))
        rpn.setdefault("num_classes", 1)
        self.rpn_head = MODELS.build(rpn)
        roi = dict(roi_head)
        roi.update(train_cfg=None, test_cfg=test_cfg.get("rcnn"))
        self.roi_head = MODELS.build(roi)
        self.shared_image_embedding = MODELS.build(shared_image_embedding)
        self.decoder_freeze = decoder_freeze
        self.test_cfg = test_cfg
        self.data_preprocessor_cfg = data_preprocessor
        self.data_preprocessor = MODELS.build(dict(data_preprocessor)) if data_preprocessor else None
        self.eval()

    @torch.no_grad()
    def predict_raw(self, batch_inputs: torch.Tensor):
        """Device-resident results: dict(bboxes [B,M,4], scores, labels, counts, mask_logits [B*M,1,4g,4g])."""
        img_hw = tuple(batch_inputs.shape[-2:])
        emb_rows, pos_rows, ghw, emb_nhwc, hidden = self._encode(batch_inputs)
        if isinstance(getattr(self.neck, "feature_aggregator", None), PseudoFeatureAggregator):
            feats = self.neck.forward_nhwc(None, _lib.cast_bf16(emb_nhwc.contiguous()))
        else:
            feats = self.neck.forward_nhwc(hidden)
        shapes = getattr(batch_inputs, "rsp_img_shapes", None)
        props, _, pcnt = self.rpn_head.predict_nhwc(feats, img_hw, img_shapes=shapes)
        return self.roi_head.predict_nhwc(feats, props, pcnt, img_hw, emb_rows, pos_rows, ghw, img_shapes=shapes)

    @torch.no_grad()
    def predict(self, batch_inputs: torch.Tensor, batch_data_samples=None, rescale: bool = True):
        if batch_data_samples is None:
            batch_data_samples = make_data_samples(batch_inputs.shape[0], tuple(batch_inputs.shape[-2:]))
        hw, metas = self._metas(batch_data_samples, batch_inputs)
        batch_inputs = self._attach_img_shapes(batch_data_samples, batch_inputs)
        r = self._raw(batch_inputs)
        if getattr(self, "_graphs", None) is not None:     # graph buffers are overwritten by the next replay
            r = dict(r, bboxes=r["bboxes"].clone(), scores=r["scores"].clone(), labels=r["labels"].clone())
        thr = float(self.test_cfg.rcnn.get("mask_thr_binary", 0.5))
        B, M = r["scores"].shape
        logits = r["mask_logits"][:, 0].contiguous()
        fast = all(m is None for m in metas)
        masks = _lib.mask_paste(logits, thr, raw=False, size=hw).view(B, M, hw[0], hw[1]) if fast else None
        counts = r["counts"].cpu().tolist()          # the only device->host read
        for b, ds in enumerate(batch_data_samples):
            n, m = counts[b], metas[b]
            boxes = r["bboxes"][b, :n]
            geom = dict(size=hw)
            if m is not None:   # resized / padded image: boxes back to the original image, masks through the two resizes
                sf, crop = m["scale_factor"], m["crop_hw"]
                if rescale:
                    boxes = boxes / boxes.new_tensor(sf).repeat(2)
                else:   # M:1756-1760 scales img_h / img_w once more before the crop; the output stays ori_shape
                    ih, iw = int(round(m["ori_hw"][0] * sf[1])), int(round(m["ori_hw"][1] * sf[0]))
                    crop = (min(int(ih * sf[1]), hw[0]), min(int(iw * sf[0]), hw[1]))
                geom = dict(rescale=(hw, crop, m["ori_hw"]))
            mk = masks[b, :n] if fast else _lib.mask_paste(logits[b * M:b * M + max(n, 1)], thr, raw=False, **geom)[:n]
            ds.pred_instances = InstanceData(bboxes=boxes, scores=r["scores"][b, :n], labels=r["labels"][b, :n], masks=mk)
        return self._rle_masks(self.test_cfg, batch_data_samples)

    @torch.no_grad()
    def predict_records(self, batch_inputs: torch.Tensor, record: ResultRecord | None = None,
                        batch_data_samples=None) -> ResultRecord:
        """predict() with the result left on the device as one ResultRecord (bit-packed masks + rows + counts): what a
        distributed test loop gathers / copies to the host.  Without samples the images are at the batch shape; with
        samples of resized images (one shared ori_shape) the rows and masks are in original-image coordinates, as
        predict(rescale=True) returns them."""
        batch_inputs, metas, rhw = self._record_metas(batch_data_samples, batch_inputs, record)
        r = self._raw(batch_inputs)
        hw = tuple(int(v) for v in batch_inputs.shape[-2:])
        B, M = r["scores"].shape
        rec = record or self._new_record(B, M, rhw or hw, r["scores"].device)
        thr = float(self.test_cfg.rcnn.get("mask_thr_binary", 0.5))
        boxes = r["bboxes"]
        if metas is None:
            _lib.mask_paste(r["mask_logits"][:, 0].contiguous(), thr, raw=False, bits=rec.mask_bits)
        else:
            logits = r["mask_logits"][:, 0].contiguous()
            for b, m in enumerate(metas):
                _lib.mask_paste(logits[b * M:(b + 1) * M], thr, raw=False, rescale=(hw, m["crop_hw"], m["ori_hw"]),
                                bits=rec.mask_bits.view(B * M, *rec.mask_bits.shape[2:])[b * M:(b + 1) * M])
            boxes = self._rescaled_boxes(boxes, metas)
        torch.cat([boxes, r["scores"][..., None], r["labels"].to(torch.float32)[..., None]], dim=2, out=rec.rows)
        rec.counts.copy_(r["counts"])
        return rec

    def forward(self, inputs, data_samples=None, mode: str = "predict"):
        if mode == "predict":
            return self.predict(inputs, data_samples)
        raise NotImplementedError("rsprompter_b200 implements the inference path only (mode='predict')")

    def test_step(self, data):
        """BaseModel.test_step: data_preprocessor(data, False) then forward(mode='predict')."""
        data = self._preprocess(data)
        return self.predict(data["inputs"], data.get("data_samples"))


@MODELS.register_module(force=True)
class RSPrompterQuery(_SamDetectorBase):
    """M:172-272 over mmdet Mask2Former / MaskFormer (detectors/maskformer.py:14-170)."""

    def __init__(self, shared_image_embedding, decoder_freeze=True, backbone=None, neck=None, panoptic_head=None,
                 panoptic_fusion_head=None, train_cfg=None, test_cfg=None, data_preprocessor=None, init_cfg=None,
                 **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        test_cfg = _cfg(test_cfg)
        self.backbone = MODELS.build(backbone)
        self.neck = MODELS.build(neck)
        ph = dict(panoptic_head)
        ph.update(train_cfg=None, test_cfg=test_cfg)
        self.panoptic_head = MODELS.build(ph)
        pf = dict(panoptic_fusion_head)
        pf.update(test_cfg=test_cfg)
        self.panoptic_fusion_head = MODELS.build(pf)
        self.shared_image_embedding = MODELS.build(shared_image_embedding)
        self.decoder_freeze = decoder_freeze
        self.test_cfg = test_cfg
        self.data_preprocessor_cfg = data_preprocessor
        self.data_preprocessor = MODELS.build(dict(data_preprocessor)) if data_preprocessor else None
        self.eval()

    @torch.no_grad()
    def predict_raw(self, batch_inputs: torch.Tensor, capture: dict | None = None):
        """-> dict(cls fp32 [B, nq, C+1], mask_logits fp32 [B*nq, 4g, 4g], mask_pred_plus fp32 [B, nq, H/4, W/4])."""
        emb_rows, pos_rows, ghw, emb_nhwc, hidden = self._encode(batch_inputs)
        if isinstance(getattr(self.neck, "feature_aggregator", None), PseudoFeatureAggregator):
            feats = self.neck.forward_nhwc(None, _lib.cast_bf16(emb_nhwc.contiguous()))
        else:
            feats = self.neck.forward_nhwc(hidden)
        cls, masks, mpp = self.panoptic_head.forward_nhwc(feats, emb_rows.contiguous(), pos_rows, ghw, capture=capture)
        return dict(cls=cls, mask_logits=masks, mask_pred_plus=mpp)

    @torch.no_grad()
    def predict(self, batch_inputs: torch.Tensor, batch_data_samples=None, rescale: bool = True):
        if batch_data_samples is None:
            batch_data_samples = make_data_samples(batch_inputs.shape[0], tuple(batch_inputs.shape[-2:]))
        hw, metas = self._metas(batch_data_samples, batch_inputs)
        # M:672-676 / maskformer_fusion_head.py:226-230 defaults; MaskFormer.add_pred_to_datasample (maskformer.py:142-148)
        if self.test_cfg.get("semantic_on", False):
            raise NotImplementedError("semantic segmentation results are not supported (as in the reference)")
        panoptic_on, instance_on = self.test_cfg.get("panoptic_on", True), self.test_cfg.get("instance_on", False)
        if panoptic_on:
            _lib.check_panoptic_bounds(self.panoptic_head.num_queries, self.panoptic_fusion_head.num_classes)
        r = self._raw(batch_inputs)
        head = self.panoptic_fusion_head
        if instance_on:
            out = head.instance_postprocess_batched(r["cls"], r["mask_logits"], hw, metas=metas, rescale=rescale)
            stuff = head.num_stuff_classes > 0
            for b, ds in enumerate(batch_data_samples):
                inst = dict(bboxes=out["bboxes"][b], scores=out["scores"][b], labels=out["labels"][b],
                            masks=out["masks"][b])
                if stuff:                                   # maskformer_fusion_head.py:160-164 (data-dependent size)
                    k = out["is_thing"][b]
                    inst = {n: v[k] for n, v in inst.items()}
                ds.pred_instances = InstanceData(**inst)
        if panoptic_on:
            pans, _ = head.panoptic_postprocess_batched(r["cls"], r["mask_logits"], hw, metas=metas, rescale=rescale)
            for ds, pan in zip(batch_data_samples, pans):
                ds.pred_panoptic_seg = PixelData(sem_seg=pan)
        return self._rle_masks(self.test_cfg, batch_data_samples)

    @torch.no_grad()
    def predict_records(self, batch_inputs: torch.Tensor, record: ResultRecord | None = None,
                        batch_data_samples=None) -> ResultRecord:
        """predict() with the result left on the device as one ResultRecord; images at the batch shape, or with
        samples of resized images (one shared ori_shape) in original-image coordinates (RSPrompterAnchor's)."""
        batch_inputs, metas, rhw = self._record_metas(batch_data_samples, batch_inputs, record)
        r = self._raw(batch_inputs)
        hw = tuple(int(v) for v in batch_inputs.shape[-2:])
        B = r["cls"].shape[0]
        K = int(self.test_cfg.get("max_per_image", 100))
        rec = record or self._new_record(B, K, rhw or hw, r["cls"].device)
        self.panoptic_fusion_head.instance_postprocess_record(r["cls"], r["mask_logits"], rec, metas=metas, size=hw)
        return rec

    def forward(self, inputs, data_samples=None, mode: str = "predict"):
        if mode == "predict":
            return self.predict(inputs, data_samples)
        raise NotImplementedError("rsprompter_b200 implements the inference path only (mode='predict')")

    def test_step(self, data):
        """BaseModel.test_step: data_preprocessor(data, False) then forward(mode='predict')."""
        data = self._preprocess(data)
        return self.predict(data["inputs"], data.get("data_samples"))


@MODELS.register_module(force=True)
class SAMSegMaskRCNN(_SamDetectorBase):
    """M:1218-1244 over mmdet MaskRCNN / TwoStageDetector.predict (detectors/two_stage.py:196-243): the SAM encoder +
    RSFPN feed the stock RPNHead -> StandardRoIHead (Shared2FCBBoxHead + FCNMaskHead); the masks are the 28x28 RoI
    masks pasted into their boxes (fcn_mask_head.py:278-418), not SAM decoder outputs."""

    def __init__(self, backbone=None, neck=None, rpn_head=None, roi_head=None, train_cfg=None, test_cfg=None,
                 data_preprocessor=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        test_cfg = _cfg(test_cfg)
        self.backbone = MODELS.build(backbone)
        self.neck = MODELS.build(neck)
        rpn = dict(rpn_head)
        rpn.update(train_cfg=None, test_cfg=test_cfg.get("rpn"))
        rpn.setdefault("num_classes", 1)
        self.rpn_head = MODELS.build(rpn)
        roi = dict(roi_head)
        roi.update(train_cfg=None, test_cfg=test_cfg.get("rcnn"))
        self.roi_head = MODELS.build(roi)
        self.test_cfg = test_cfg
        self.data_preprocessor_cfg = data_preprocessor
        self.data_preprocessor = MODELS.build(dict(data_preprocessor)) if data_preprocessor else None
        self.eval()

    def extract_feat(self, batch_inputs: torch.Tensor):
        """M:1233-1244: the neck outputs only (NCHW tuple)."""
        vision_outputs = self.backbone(batch_inputs)
        if isinstance(vision_outputs, SamVisionEncoderOutput):
            hidden = vision_outputs[1]
        elif isinstance(vision_outputs, tuple):
            hidden = vision_outputs
        else:
            raise NotImplementedError
        return self.neck(hidden)

    @torch.no_grad()
    def predict_raw(self, batch_inputs: torch.Tensor, capture: dict | None = None):
        """Device-resident results: dict(bboxes [B,M,4], scores, labels, counts, mask_probs fp32 [B*M, 28, 28])."""
        img_hw = tuple(batch_inputs.shape[-2:])
        _, _, _, emb_nhwc, hidden = self._encode(batch_inputs)
        if isinstance(getattr(self.neck, "feature_aggregator", None), PseudoFeatureAggregator):
            feats = self.neck.forward_nhwc(None, _lib.cast_bf16(emb_nhwc.contiguous()))
        else:
            feats = self.neck.forward_nhwc(hidden)
        shapes = getattr(batch_inputs, "rsp_img_shapes", None)
        props, _, pcnt = self.rpn_head.predict_nhwc(feats, img_hw, img_shapes=shapes)
        if capture is not None:
            capture.update(feats=feats, proposals=props, prop_counts=pcnt)
        return self.roi_head.predict_nhwc(feats, props, pcnt, img_hw, capture=capture, img_shapes=shapes)

    @torch.no_grad()
    def predict(self, batch_inputs: torch.Tensor, batch_data_samples=None, rescale: bool = True):
        if batch_data_samples is None:
            batch_data_samples = make_data_samples(batch_inputs.shape[0], tuple(batch_inputs.shape[-2:]))
        hw, metas = self._metas(batch_data_samples, batch_inputs)
        batch_inputs = self._attach_img_shapes(batch_data_samples, batch_inputs)
        r = self._raw(batch_inputs)
        if getattr(self, "_graphs", None) is not None:     # graph buffers are overwritten by the next replay
            r = {k: v.clone() for k, v in r.items()}
        thr = float(self.test_cfg.rcnn.get("mask_thr_binary", 0.5))
        B, M = r["scores"].shape
        probs = r["mask_probs"]
        fast = all(m is None for m in metas)
        masks = _lib.mask_paste_boxes(probs, r["bboxes"].reshape(B * M, 4), hw, thr).view(B, M, *hw) if fast else None
        counts = r["counts"].cpu().tolist()          # the only device->host read
        for b, ds in enumerate(batch_data_samples):
            n, m = counts[b], metas[b]
            boxes = r["bboxes"][b, :n]
            if fast:
                mk = masks[b, :n]
            else:   # fcn_mask_head.py:333-343: boxes to the original image (rescale) or canvas = round(ori * scale)
                size = hw
                if m is not None:
                    sf, size = m["scale_factor"], m["ori_hw"]
                    if rescale:
                        boxes = boxes / boxes.new_tensor(sf).repeat(2)
                    else:
                        size = (int(round(size[0] * sf[1])), int(round(size[1] * sf[0])))
                pb = torch.zeros(max(n, 1), 4, device=boxes.device)
                pb[:n] = boxes
                mk = _lib.mask_paste_boxes(probs[b * M:b * M + max(n, 1)].contiguous(), pb, size, thr)[:n]
            ds.pred_instances = InstanceData(bboxes=boxes, scores=r["scores"][b, :n], labels=r["labels"][b, :n], masks=mk)
        return self._rle_masks(self.test_cfg, batch_data_samples)

    @torch.no_grad()
    def predict_records(self, batch_inputs: torch.Tensor, record: ResultRecord | None = None,
                        batch_data_samples=None) -> ResultRecord:
        """predict() left on the device as one ResultRecord; images at the batch shape, or with samples of resized
        images (one shared ori_shape) in original-image coordinates: the RoI masks are pasted into the rescaled boxes
        on the record's canvas (fcn_mask_head.py:333-343), which agrees with predict() on ori_shape."""
        batch_inputs, metas, rhw = self._record_metas(batch_data_samples, batch_inputs, record)
        r = self._raw(batch_inputs)
        hw = tuple(int(v) for v in batch_inputs.shape[-2:])
        B, M = r["scores"].shape
        rec = record or self._new_record(B, M, rhw or hw, r["scores"].device)
        thr = float(self.test_cfg.rcnn.get("mask_thr_binary", 0.5))
        boxes = r["bboxes"]
        if metas is not None:
            boxes = self._rescaled_boxes(boxes, metas)
        _lib.mask_paste_boxes(r["mask_probs"], boxes.reshape(B * M, 4).contiguous(), rec.hw, thr, bits=rec.mask_bits)
        torch.cat([boxes, r["scores"][..., None], r["labels"].to(torch.float32)[..., None]], dim=2, out=rec.rows)
        rec.counts.copy_(r["counts"])
        return rec

    def forward(self, inputs, data_samples=None, mode: str = "predict"):
        if mode == "predict":
            return self.predict(inputs, data_samples)
        raise NotImplementedError("rsprompter_b200 implements the inference path only (mode='predict')")

    def test_step(self, data):
        data = self._preprocess(data)
        return self.predict(data["inputs"], data.get("data_samples"))


@MODELS.register_module(force=True)
class SAMSegMask2Former(_SamDetectorBase):
    """M:1247-1274 over mmdet Mask2Former / MaskFormer.predict (detectors/maskformer.py:95-140): SAM encoder + RSFPN
    feed the stock Mask2FormerHead; MaskFormerFusionHead turns the last layer's (cls, masks) into instances."""

    def __init__(self, backbone=None, neck=None, panoptic_head=None, panoptic_fusion_head=None, train_cfg=None,
                 test_cfg=None, data_preprocessor=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        test_cfg = _cfg(test_cfg)
        self.backbone = MODELS.build(backbone)
        self.neck = MODELS.build(neck)
        ph = dict(panoptic_head)
        ph.update(train_cfg=None, test_cfg=test_cfg)
        self.panoptic_head = MODELS.build(ph)
        pf = dict(panoptic_fusion_head)
        pf.update(test_cfg=test_cfg)
        self.panoptic_fusion_head = MODELS.build(pf)
        self.test_cfg = test_cfg
        self.data_preprocessor_cfg = data_preprocessor
        self.data_preprocessor = MODELS.build(dict(data_preprocessor)) if data_preprocessor else None
        self.eval()

    extract_feat = SAMSegMaskRCNN.extract_feat

    @torch.no_grad()
    def predict_raw(self, batch_inputs: torch.Tensor, capture: dict | None = None):
        """-> dict(cls fp32 [B, nq, C+1], mask_logits fp32 [B*nq, H/4, W/4])."""
        _, _, _, emb_nhwc, hidden = self._encode(batch_inputs)
        if isinstance(getattr(self.neck, "feature_aggregator", None), PseudoFeatureAggregator):
            feats = self.neck.forward_nhwc(None, _lib.cast_bf16(emb_nhwc.contiguous()))
        else:
            feats = self.neck.forward_nhwc(hidden)
        if capture is not None:
            capture.update(feats=feats)
        cls, masks = self.panoptic_head.forward_nhwc(feats, capture=capture)
        return dict(cls=cls, mask_logits=masks)

    predict = RSPrompterQuery.predict
    predict_records = RSPrompterQuery.predict_records
    forward = RSPrompterQuery.forward
    test_step = RSPrompterQuery.test_step


__all__ = ["RSPrompterAnchor", "RSPrompterQuery", "SAMSegMaskRCNN", "SAMSegMask2Former"]
