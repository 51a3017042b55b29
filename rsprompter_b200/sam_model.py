"""Box-prompted SAM on the H100 kernels: ``RSSamModel`` (M:718-741 over HF ``SamModel``, HF:1075-1300) and the
``SAMDet`` detector that prompts it with another detector's boxes (M:1060-1215) - SURVEY 8(f4).

``RSSamModel.sam_model`` keeps HF ``SamModel``'s parameter tree (``vision_encoder.*``, ``prompt_encoder.*``,
``mask_decoder.*``, ``shared_image_embedding.positional_embedding``), so ``facebook/sam-vit-*`` checkpoints load
unchanged.  The forward is the encoder of ``sam_encoder.py`` and the decoder of ``sam_decoder.py`` with the prompts of
one image sharing its embedding through block maps; the prompt encoder's box path (HF ``_embed_boxes``: two corner
points through the random-Fourier positional embedding + ``point_embed[2|3]``) is a handful of elementwise device ops
on [B, n_boxes, 2, 2] coordinates."""
from __future__ import annotations

from collections import OrderedDict

import torch
from torch import nn

from . import _lib
from .registry import MODELS, BaseModule, ConfigDict, InstanceData
from .sam_config import decoder_arch, vision_arch
from .sam_decoder import SamMaskDecoderB200, SamPositionalEmbeddingB200, _Embedding, _MaskEmbed
from .sam_encoder import SamVisionEncoderB200, _load_pretrained


class SamImageSegmentationOutput(OrderedDict):
    """(iou_scores, pred_masks) with attribute access, like HF's ModelOutput of the same name."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class _PromptEncoder(nn.Module):
    """HF SamPromptEncoder parameter tree (HF:596-611)."""

    def __init__(self, va, da):
        super().__init__()
        self.shared_embedding = SamPositionalEmbeddingB200(va.num_pos_feats, va.pe_scale())
        self.mask_embed = _MaskEmbed(da)
        self.no_mask_embed = _Embedding(1, da.hidden_size)
        self.point_embed = nn.ModuleList(_Embedding(1, da.hidden_size) for _ in range(4))
        self.not_a_point_embed = _Embedding(1, da.hidden_size)


class SamModelB200(nn.Module):
    def __init__(self, va, da):
        super().__init__()
        self.varch, self.darch = va, da
        self.shared_image_embedding = SamPositionalEmbeddingB200(va.num_pos_feats, va.pe_scale())
        self.vision_encoder = SamVisionEncoderB200(va)
        self.prompt_encoder = _PromptEncoder(va, da)
        self.mask_decoder = SamMaskDecoderB200(da)
        # HF ties prompt_encoder.shared_embedding to shared_image_embedding: checkpoints carry one or both names
        self._register_load_state_dict_pre_hook(self._tie_shared_embedding)

    @staticmethod
    def _tie_shared_embedding(state_dict, prefix, *args):
        a, b = prefix + "shared_image_embedding.positional_embedding", prefix + "prompt_encoder.shared_embedding.positional_embedding"
        if a in state_dict and b not in state_dict:
            state_dict[b] = state_dict[a]
        elif b in state_dict and a not in state_dict:
            state_dict[a] = state_dict[b]

    def embed_boxes(self, boxes: torch.Tensor) -> torch.Tensor:
        """HF SamPromptEncoder._embed_boxes: [B, nb, 4] image-space xyxy -> sparse embeddings [B, nb, 2, C]."""
        pe = self.prompt_encoder
        S = self.varch.image_size
        coords = (boxes.to(torch.float32) + 0.5).reshape(*boxes.shape[:2], 2, 2)
        emb = pe.shared_embedding(coords, (S, S))
        corner = torch.stack([pe.point_embed[2].weight[0], pe.point_embed[3].weight[0]]).to(emb.dtype)
        return emb + corner.view(1, 1, 2, -1)

    @torch.no_grad()
    def forward(self, pixel_values=None, input_points=None, input_labels=None, input_boxes=None, input_masks=None,
                image_embeddings=None, multimask_output: bool = True, attention_similarity=None, target_embedding=None,
                **kwargs):
        if pixel_values is None and image_embeddings is None:
            raise ValueError("Either pixel_values or image_embeddings must be provided.")
        if pixel_values is not None and image_embeddings is not None:
            raise ValueError("Only one of pixel_values and image_embeddings can be provided.")
        if input_boxes is None or input_points is not None or input_masks is not None:
            raise NotImplementedError("rsprompter_b200 RSSamModel implements the box-prompted path SAMDet uses (M:1120-1131)")
        if input_boxes.dim() != 3:
            raise ValueError(f"The input_points must be a 3D tensor. Of shape `batch_size`, `nb_boxes`, `4`. got {input_boxes.shape}.")
        if attention_similarity is not None or target_embedding is not None:
            raise NotImplementedError("attention_similarity / target_embedding are not used by RSPrompter")
        C = self.darch.hidden_size
        if pixel_values is not None:
            _, _, emb_nhwc = self.vision_encoder.encode(pixel_values, want_hidden=False)
        else:
            emb_nhwc = image_embeddings.to(torch.float32).permute(0, 2, 3, 1).contiguous()
        B, g = emb_nhwc.shape[0], emb_nhwc.shape[1]
        nb = input_boxes.shape[1]
        assert input_boxes.shape[0] == B
        sparse = self.embed_boxes(input_boxes.to(emb_nhwc.device)).reshape(B * nb, 2, C).contiguous()
        prompt_img = torch.arange(B, device=emb_nhwc.device, dtype=torch.int32).repeat_interleave(nb).contiguous()
        pos_rows = self.shared_image_embedding.image_wide_rows(g)
        dense = self.prompt_encoder.no_mask_embed.weight[0].to(torch.float32).contiguous()
        masks, iou = self.mask_decoder.decode(emb_nhwc.reshape(B * g * g, C), pos_rows, sparse, (g, g),
                                              prompt_img=prompt_img, dense_vec=dense, multimask_output=multimask_output)
        return SamImageSegmentationOutput(iou_scores=iou.view(B, nb, -1),
                                          pred_masks=masks.view(B, nb, masks.shape[1], *masks.shape[-2:]))


@MODELS.register_module(force=True)
class RSSamModel(BaseModule):
    """Drop-in for mmdet.rsprompter RSSamModel (M:718-741)."""

    def __init__(self, hf_pretrain_name, extra_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        self.sam_model = SamModelB200(vision_arch(hf_pretrain_name, (extra_config or {}).get("vision_config")),
                                      decoder_arch(hf_pretrain_name, (extra_config or {}).get("mask_decoder_config")))
        _load_pretrained(self.sam_model, init_cfg, [(r"^module\.", "")])
        self.sam_model.is_init = True

    def init_weights(self):
        pass

    def forward(self, *args, **kwargs):
        return self.sam_model(*args, **kwargs)


@MODELS.register_module(force=True)
class SAMDet(BaseModule):
    """M:1060-1215: boxes from ``detector`` (or the ground truth with test_cfg.oracle_on, the reference's default)
    prompt the SAM ``segmentor``; masks go low-res logits -> img_shape -> crop to the resized image -> ori_shape -> > 0
    in one fused kernel per image (rsp_mask_paste_rescale, no intermediate maps)."""

    def __init__(self, detector, segmentor, data_preprocessor=None, test_cfg=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        self.detector = MODELS.build(detector)
        self.segmentor = MODELS.build(segmentor)
        self.segmentor.eval()
        self.test_cfg = ConfigDict(test_cfg) if isinstance(test_cfg, dict) else test_cfg
        self.data_preprocessor = MODELS.build(dict(data_preprocessor)) if data_preprocessor else None
        self.eval()

    def extract_feat(self, batch_inputs):
        pass

    @torch.no_grad()
    def _segment(self, input_img: torch.Tensor, bboxes: torch.Tensor, meta: dict) -> torch.Tensor:
        ori_h, ori_w = (int(v) for v in meta["ori_shape"][:2])
        if bboxes.shape[0] == 0:
            return torch.zeros(0, ori_h, ori_w, device=input_img.device, dtype=torch.bool)
        sf = tuple(float(s) for s in meta.get("scale_factor", (1.0, 1.0)))
        boxes = bboxes * bboxes.new_tensor(sf).repeat((1, bboxes.size(-1) // 2))
        out = self.segmentor(pixel_values=input_img.unsqueeze(0), input_boxes=boxes.unsqueeze(0), multimask_output=False)
        logits = out.pred_masks[0][:, 0].contiguous()                     # [nb, 4g, 4g]
        img_hw = tuple(int(v) for v in meta["img_shape"][:2])
        crop = (min(int(ori_h * sf[1]), img_hw[0]), min(int(ori_w * sf[0]), img_hw[1]))
        return _lib.mask_paste_rescale(logits, img_hw, crop, (ori_h, ori_w), 0.0, raw=True)

    @torch.no_grad()
    def predict(self, batch_inputs, batch_data_samples, rescale: bool = True):
        oracle = self.test_cfg is not None and self.test_cfg.get("oracle_on", True)
        batch_data_samples = self.detector.predict(batch_inputs, batch_data_samples, rescale=rescale)
        for input_img, ds in zip(batch_inputs, batch_data_samples):
            if oracle:                                                   # M:1091-1097: ground-truth boxes as prompts
                gt = ds.gt_instances
                inst = InstanceData(bboxes=gt.bboxes, labels=gt.labels,
                                    scores=torch.ones_like(gt.labels, dtype=torch.float32))
            else:
                inst = ds.pred_instances
            inst.masks = self._segment(input_img, inst.bboxes.to(input_img.device), ds.metainfo)
            ds.pred_instances = inst
        return batch_data_samples

    def forward(self, inputs, data_samples=None, mode: str = "predict"):
        if mode == "predict":
            return self.predict(inputs, data_samples)
        raise NotImplementedError("rsprompter_b200 implements the inference path only (mode='predict')")

    def test_step(self, data):
        if self.data_preprocessor is not None:
            data = self.data_preprocessor(data, False)
        return self.predict(data["inputs"], data.get("data_samples"))


__all__ = ["SamModelB200", "RSSamModel", "SAMDet", "SamImageSegmentationOutput"]
