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
from .sam_decoder import SamMaskDecoderB200, SamPositionalEmbeddingB200, _Embedding, _MaskEmbed, check_sparse_tokens
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

    def embed_points(self, points: torch.Tensor, labels: torch.Tensor, pad: bool) -> torch.Tensor:
        """HF SamPromptEncoder._embed_points (HF:613-645): [B, pb, n, 2] image-space xy and [B, pb, n] labels ->
        sparse embeddings [B, pb, n (+1 with pad), C].  Label -1: not_a_point_embed; -10: zero; 0 / 1: + point_embed[0
        / 1]; any other label keeps the bare positional embedding."""
        pe = self.prompt_encoder
        S = self.varch.image_size
        coords = points.to(torch.float32) + 0.5
        if pad:
            coords = torch.cat([coords, coords.new_zeros(*coords.shape[:2], 1, 2)], dim=2)
            labels = torch.cat([labels, labels.new_full((*labels.shape[:2], 1), -1)], dim=2)
        emb = pe.shared_embedding(coords, (S, S))
        lab = labels[..., None]
        emb = torch.where(lab == -1, pe.not_a_point_embed.weight[0].to(emb.dtype), emb)
        emb = torch.where(lab != -10, emb, torch.zeros_like(emb))
        emb = torch.where(lab == 0, emb + pe.point_embed[0].weight[0].to(emb.dtype), emb)
        return torch.where(lab == 1, emb + pe.point_embed[1].weight[0].to(emb.dtype), emb)

    def _check_prompts(self, n_images, input_points, input_labels, input_boxes, input_masks, grid: int) -> tuple:
        """HF SamModel.forward's shape rules (HF:1286-1334) plus the token bound of the decoder kernels, all before any
        device work.  -> (point_batch, sparse tokens per prompt)."""
        if input_points is not None and input_points.dim() != 4:
            raise ValueError("The input_points must be a 4D tensor. Of shape `batch_size`, `point_batch_size`, "
                             f"`nb_points_per_image`, `2`. got {tuple(input_points.shape)}.")
        if input_points is not None and input_points.shape[-1] != 2:
            raise ValueError(f"input_points must hold (x, y) pairs, got last dimension {input_points.shape[-1]}")
        if input_boxes is not None and (input_boxes.dim() != 3 or input_boxes.shape[-1] != 4):
            raise ValueError("The input_boxes must be a 3D tensor. Of shape `batch_size`, `nb_boxes`, `4`. "
                             f"got {tuple(input_boxes.shape)}.")
        if input_points is not None and input_boxes is not None and input_points.shape[1] != input_boxes.shape[1]:
            raise ValueError("You should provide as many bounding boxes as input points per box. "
                             f"Got {input_points.shape[1]} and {input_boxes.shape[1]}.")
        for name, t in (("input points", input_points), ("input boxes", input_boxes)):
            if t is not None and t.shape[0] != n_images:
                raise ValueError(f"The batch size of the image embeddings and the {name} must be the same. "
                                 f"Got {n_images} and {t.shape[0]} respectively.")
        if input_labels is not None and input_points is not None and tuple(input_labels.shape) != tuple(input_points.shape[:3]):
            raise ValueError(f"input_labels must be [batch, point_batch, n_points] like input_points[..., 0], got "
                             f"{tuple(input_labels.shape)}")
        if input_masks is not None and tuple(input_masks.shape) != (n_images, 1, 4 * grid, 4 * grid):
            raise ValueError(f"input_masks must be [{n_images}, 1, {4 * grid}, {4 * grid}], got {tuple(input_masks.shape)}")
        pb, P = 1, 0
        if input_points is not None:
            pb, P = input_points.shape[1], input_points.shape[2] + (1 if input_boxes is None else 0)
        if input_boxes is not None:
            pb, P = input_boxes.shape[1], P + 2
        check_sparse_tokens(P, self.mask_decoder.num_mask_tokens)
        return pb, P

    def _sparse(self, input_points, input_labels, input_boxes, dev) -> torch.Tensor | None:
        """sparse = cat([points (no pad point when boxes are given), box corners], dim=2) (HF:676-690)."""
        parts = []
        if input_points is not None:
            if input_labels is None:
                input_labels = torch.ones(input_points.shape[:3], dtype=torch.int32)
            parts.append(self.embed_points(input_points.to(dev), input_labels.to(dev), pad=input_boxes is None))
        if input_boxes is not None:
            parts.append(self.embed_boxes(input_boxes.to(dev)))
        if not parts:
            return None
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=2)

    def _encode(self, pixel_values) -> torch.Tensor:
        _, _, emb_nhwc = self.vision_encoder.encode(pixel_values, want_hidden=False)
        return emb_nhwc

    @torch.no_grad()
    def get_image_embeddings(self, pixel_values) -> torch.Tensor:
        """HF SamModel.get_image_embeddings (HF:1142-1155): fp32 [B, 256, g, g].  Passing them back as
        forward(image_embeddings=...) gives the bytes of forward(pixel_values=...)."""
        return self._encode(pixel_values).permute(0, 3, 1, 2)

    @torch.no_grad()
    def get_prompt_embeddings(self, input_points=None, input_labels=None, input_boxes=None, input_masks=None):
        """HF SamModel.get_prompt_embeddings (HF:1158-1191) -> (sparse [B, pb, P, 256] or None, dense [B, 256, g, g]);
        without a mask prompt dense is no_mask_embed broadcast over the batch of the sparse prompts (1 if none)."""
        if input_points is not None and input_labels is None:
            raise ValueError("If points are provided, labels must also be provided.")
        g = self.varch.grid
        n = next((t.shape[0] for t in (input_points, input_boxes, input_masks) if t is not None), 1)
        self._check_prompts(n, input_points, input_labels, input_boxes, input_masks, g)
        dev = self.prompt_encoder.no_mask_embed.weight.device
        sparse = self._sparse(input_points, input_labels, input_boxes, dev)
        C = self.darch.hidden_size
        if input_masks is not None:
            rows = self.prompt_encoder.mask_embed.dense_rows(input_masks, self.darch.layer_norm_eps)
            return sparse, rows.view(n, g, g, C).permute(0, 3, 1, 2)
        return sparse, self.prompt_encoder.no_mask_embed.weight.reshape(1, -1, 1, 1).expand(n, -1, g, g)

    @torch.no_grad()
    def forward(self, pixel_values=None, input_points=None, input_labels=None, input_boxes=None, input_masks=None,
                image_embeddings=None, multimask_output: bool = True, attention_similarity=None, target_embedding=None,
                **kwargs):
        """HF SamModel.forward (HF:1193-1358): points [B, pb, n, 2] with labels [B, pb, n] (None: all 1), boxes
        [B, pb, 4], points and boxes together, a low-res mask prompt [B, 1, 4g, 4g], pixel_values or image_embeddings.
        -> iou_scores [B, pb, n_out], pred_masks [B, pb, n_out, 4g, 4g]."""
        if pixel_values is None and image_embeddings is None:
            raise ValueError("Either pixel_values or image_embeddings must be provided.")
        if pixel_values is not None and image_embeddings is not None:
            raise ValueError("Only one of pixel_values and image_embeddings can be provided.")
        if attention_similarity is not None or target_embedding is not None:
            raise NotImplementedError("attention_similarity / target_embedding are not used by RSPrompter")
        n_images = pixel_values.shape[0] if pixel_values is not None else image_embeddings.shape[0]
        grid = self.varch.grid if pixel_values is not None else image_embeddings.shape[-1]
        pb, _ = self._check_prompts(n_images, input_points, input_labels, input_boxes, input_masks, grid)
        C = self.darch.hidden_size
        if pixel_values is not None:
            emb_nhwc = self._encode(pixel_values)
        else:
            emb_nhwc = image_embeddings.to(torch.float32).permute(0, 2, 3, 1).contiguous()
        B, g = emb_nhwc.shape[0], emb_nhwc.shape[1]
        dev = emb_nhwc.device
        if input_points is None and input_masks is None and input_boxes is not None:
            # boxes only (SAMDet, M:1120-1131)
            nb = input_boxes.shape[1]
            sparse = self.embed_boxes(input_boxes.to(dev)).reshape(B * nb, 2, C).contiguous()
            prompt_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(nb).contiguous()
            pos_rows = self.shared_image_embedding.image_wide_rows(g)
            dense = self.prompt_encoder.no_mask_embed.weight[0].to(torch.float32).contiguous()
            masks, iou = self.mask_decoder.decode(emb_nhwc.reshape(B * g * g, C), pos_rows, sparse, (g, g),
                                                  prompt_img=prompt_img, dense_vec=dense,
                                                  multimask_output=multimask_output)
            return SamImageSegmentationOutput(iou_scores=iou.view(B, nb, -1),
                                              pred_masks=masks.view(B, nb, masks.shape[1], *masks.shape[-2:]))
        sparse = self._sparse(input_points, input_labels, input_boxes, dev)
        if sparse is None:                 # no sparse prompt: the 5 output tokens alone (HF:487-495)
            sparse = emb_nhwc.new_zeros(B, 1, 0, C)
        P = sparse.shape[2]
        sparse = sparse.reshape(B * pb, P, C).contiguous()
        prompt_img = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(pb).contiguous()
        pos_rows = self.shared_image_embedding.image_wide_rows(g)
        emb_rows = emb_nhwc.reshape(B * g * g, C)
        if input_masks is not None:        # one dense term per image (HF:499-500), shared by its prompts
            dense_img = self.prompt_encoder.mask_embed.dense_rows(input_masks, self.darch.layer_norm_eps)
            masks, iou = self.mask_decoder.decode(emb_rows, pos_rows, sparse, (g, g), prompt_img=prompt_img,
                                                  dense_img_rows=dense_img, multimask_output=multimask_output)
        else:
            dense = self.prompt_encoder.no_mask_embed.weight[0].to(torch.float32).contiguous()
            masks, iou = self.mask_decoder.decode(emb_rows, pos_rows, sparse, (g, g), prompt_img=prompt_img,
                                                  dense_vec=dense, multimask_output=multimask_output)
        return SamImageSegmentationOutput(iou_scores=iou.view(B, pb, -1),
                                          pred_masks=masks.view(B, pb, masks.shape[1], *masks.shape[-2:]))


@torch.no_grad()
def post_process_masks(masks, original_sizes, reshaped_input_sizes, mask_threshold: float = 0.0,
                       binarize: bool = True, pad_size=(1024, 1024)) -> list:
    """HF SamProcessor.post_process_masks on the device: per image, low-res logits [pb, n_out, h, w] -> bilinear to
    pad_size -> crop to the reshaped (resized, unpadded) input size -> bilinear to the original size -> > threshold, in
    one fused kernel (rsp_mask_paste through two resizes, the SAMDet path).  -> list of bool [pb, n_out, H, W]."""
    if not binarize:
        raise ValueError("post_process_masks computes binary masks only (binarize=False is not supported)")
    if len(original_sizes) != len(masks) or len(reshaped_input_sizes) != len(masks):
        raise ValueError("masks, original_sizes and reshaped_input_sizes need one entry per image")
    out = []
    for m, ori, rs in zip(masks, original_sizes, reshaped_input_sizes):
        ori = tuple(int(v) for v in ori)
        rs = tuple(int(v) for v in rs)
        lead = m.shape[:-2]
        logits = m.reshape(-1, *m.shape[-2:]).to(torch.float32).contiguous()
        if logits.shape[0] == 0:
            out.append(torch.zeros(*lead, *ori, dtype=torch.bool, device=m.device))
            continue
        bits = _lib.mask_paste(logits, float(mask_threshold), raw=True, rescale=(tuple(int(v) for v in pad_size), rs, ori))
        out.append(bits.view(*lead, *ori))
    return out


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

    def get_image_embeddings(self, pixel_values):
        return self.sam_model.get_image_embeddings(pixel_values)

    def get_prompt_embeddings(self, input_points=None, input_labels=None, input_boxes=None, input_masks=None):
        return self.sam_model.get_prompt_embeddings(input_points, input_labels, input_boxes, input_masks)

    def generate_masks(self, images=None, **kwargs) -> list:
        """Segment everything: HF's mask-generation pipeline with one crop layer (see mask_generation.generate_masks)."""
        from .mask_generation import generate_masks
        return generate_masks(self, images, **kwargs)

    def generate_scene_masks(self, scene, **kwargs) -> dict:
        """Segment everything in a whole scene, window by window (see mask_generation.generate_scene_masks)."""
        from .mask_generation import generate_scene_masks
        return generate_scene_masks(self, scene, **kwargs)


@MODELS.register_module(force=True)
class SAMDet(BaseModule):
    """M:1060-1215: boxes from ``detector`` (or the ground truth with test_cfg.oracle_on, the reference's default)
    prompt the SAM ``segmentor``; masks go low-res logits -> img_shape -> crop to the resized image -> ori_shape -> > 0
    in one fused kernel per image (rsp_mask_paste through two resizes, no intermediate maps)."""

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
        return _lib.mask_paste(logits, 0.0, raw=True, rescale=(img_hw, crop, (ori_h, ori_w)))

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
        from .detectors import _SamDetectorBase
        return _SamDetectorBase._rle_masks(self.test_cfg, batch_data_samples)

    def forward(self, inputs, data_samples=None, mode: str = "predict"):
        if mode == "predict":
            return self.predict(inputs, data_samples)
        raise NotImplementedError("rsprompter_b200 implements the inference path only (mode='predict')")

    def test_step(self, data):
        if self.data_preprocessor is not None:
            data = self.data_preprocessor(data, False)
        return self.predict(data["inputs"], data.get("data_samples"))


__all__ = ["SamModelB200", "RSSamModel", "SAMDet", "SamImageSegmentationOutput", "post_process_masks"]
