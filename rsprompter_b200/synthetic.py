"""Seeded random checkpoints with the reference's parameter names and shapes.

No SAM / RSPrompter weights exist offline, so benchmarks and parity tests run on random
weights of the exact architecture (SURVEY.md appendix A; HF ``pytorch_model.bin`` key names
with the ``vision_encoder.`` prefix stripped as M:783 does).  Relative-position tables and the
absolute position embedding are drawn non-zero (HF zero-initialises them, HF:1008-1014, which
would hide every rel-pos bug).  The same dicts are loaded into the oracle (HF modules /
restatement) and into the H100 modules, so parity compares arithmetic, not initialisation.
"""
from __future__ import annotations

import math

import torch

from .sam_config import SamDecoderArch, SamVisionArch


def _randn(gen: torch.Generator, *shape: int, std: float = 0.02) -> torch.Tensor:
    return torch.randn(*shape, generator=gen, dtype=torch.float32) * std


def _linear(sd: dict, gen: torch.Generator, prefix: str, out_f: int, in_f: int, bias: bool = True,
            std: float | None = None) -> None:
    std = std if std is not None else 1.0 / math.sqrt(in_f)
    sd[prefix + ".weight"] = _randn(gen, out_f, in_f, std=std)
    if bias:
        sd[prefix + ".bias"] = _randn(gen, out_f, std=0.02)


def _norm(sd: dict, gen: torch.Generator, prefix: str, c: int) -> None:
    sd[prefix + ".weight"] = 1.0 + _randn(gen, c, std=0.05)
    sd[prefix + ".bias"] = _randn(gen, c, std=0.05)


def vision_encoder_state_dict(arch: SamVisionArch, seed: int = 0) -> dict[str, torch.Tensor]:
    """Keys of HF ``SamVisionEncoder`` (= RSSamVisionEncoder.vision_encoder.*)."""
    gen = torch.Generator().manual_seed(seed)
    D, hd, g = arch.hidden_size, arch.head_dim, arch.grid
    sd: dict[str, torch.Tensor] = {}
    sd["pos_embed"] = _randn(gen, 1, g, g, D, std=0.02)
    sd["patch_embed.projection.weight"] = _randn(gen, D, 3, arch.patch_size, arch.patch_size,
                                                 std=1.0 / math.sqrt(3 * arch.patch_size ** 2))
    sd["patch_embed.projection.bias"] = _randn(gen, D, std=0.02)
    for i in range(arch.num_layers):
        p = f"layers.{i}."
        S = g if i in arch.global_attn_indexes else arch.window_size
        _norm(sd, gen, p + "layer_norm1", D)
        sd[p + "attn.rel_pos_h"] = _randn(gen, 2 * S - 1, hd, std=0.1)
        sd[p + "attn.rel_pos_w"] = _randn(gen, 2 * S - 1, hd, std=0.1)
        _linear(sd, gen, p + "attn.qkv", 3 * D, D)
        _linear(sd, gen, p + "attn.proj", D, D, std=0.5 / math.sqrt(D))
        _norm(sd, gen, p + "layer_norm2", D)
        _linear(sd, gen, p + "mlp.lin1", arch.mlp_dim, D)
        _linear(sd, gen, p + "mlp.lin2", D, arch.mlp_dim, std=0.5 / math.sqrt(arch.mlp_dim))
    C = arch.output_channels
    sd["neck.conv1.weight"] = _randn(gen, C, D, 1, 1, std=1.0 / math.sqrt(D))
    _norm(sd, gen, "neck.layer_norm1", C)
    sd["neck.conv2.weight"] = _randn(gen, C, C, 3, 3, std=1.0 / math.sqrt(9 * C))
    _norm(sd, gen, "neck.layer_norm2", C)
    return sd


def mask_decoder_state_dict(arch: SamDecoderArch | None = None, seed: int = 1) -> dict[str, torch.Tensor]:
    """Keys of HF ``SamMaskDecoder`` (= RSSamMaskDecoder.mask_decoder.*)."""
    arch = arch or SamDecoderArch()
    gen = torch.Generator().manual_seed(seed)
    C = arch.hidden_size
    sd: dict[str, torch.Tensor] = {}
    sd["iou_token.weight"] = _randn(gen, 1, C, std=0.5)
    sd["mask_tokens.weight"] = _randn(gen, arch.num_multimask_outputs + 1, C, std=0.5)

    def attn(prefix: str, internal: int) -> None:
        for n in ("q_proj", "k_proj", "v_proj"):
            _linear(sd, gen, f"{prefix}.{n}", internal, C)
        _linear(sd, gen, f"{prefix}.out_proj", C, internal)

    for i in range(arch.num_layers):
        p = f"transformer.layers.{i}."
        attn(p + "self_attn", C)
        attn(p + "cross_attn_token_to_image", C // arch.attention_downsample_rate)
        attn(p + "cross_attn_image_to_token", C // arch.attention_downsample_rate)
        _linear(sd, gen, p + "mlp.lin1", arch.mlp_dim, C)
        _linear(sd, gen, p + "mlp.lin2", C, arch.mlp_dim)
        for k in range(1, 5):
            _norm(sd, gen, p + f"layer_norm{k}", C)
    attn("transformer.final_attn_token_to_image", C // arch.attention_downsample_rate)
    _norm(sd, gen, "transformer.layer_norm_final_attn", C)
    sd["upscale_conv1.weight"] = _randn(gen, C, C // 4, 2, 2, std=1.0 / math.sqrt(C))
    sd["upscale_conv1.bias"] = _randn(gen, C // 4, std=0.02)
    _norm(sd, gen, "upscale_layer_norm", C // 4)
    sd["upscale_conv2.weight"] = _randn(gen, C // 4, C // 8, 2, 2, std=1.0 / math.sqrt(C // 4))
    sd["upscale_conv2.bias"] = _randn(gen, C // 8, std=0.02)
    for i in range(arch.num_multimask_outputs + 1):
        p = f"output_hypernetworks_mlps.{i}."
        _linear(sd, gen, p + "proj_in", C, C)
        _linear(sd, gen, p + "layers.0", C, C)
        _linear(sd, gen, p + "proj_out", C // 8, C)
    _linear(sd, gen, "iou_prediction_head.proj_in", arch.iou_head_hidden_dim, C)
    for k in range(arch.iou_head_depth - 2):
        _linear(sd, gen, f"iou_prediction_head.layers.{k}", arch.iou_head_hidden_dim, arch.iou_head_hidden_dim)
    _linear(sd, gen, "iou_prediction_head.proj_out", arch.num_multimask_outputs + 1, arch.iou_head_hidden_dim)
    return sd


def prompt_encoder_state_dict(arch: SamDecoderArch | None = None, seed: int = 2) -> dict[str, torch.Tensor]:
    """The members of HF ``SamPromptEncoder`` the path uses (M:305-307,1635): no_mask_embed, mask_embed."""
    arch = arch or SamDecoderArch()
    gen = torch.Generator().manual_seed(seed)
    C, mc = arch.hidden_size, arch.mask_input_channels
    sd: dict[str, torch.Tensor] = {}
    sd["no_mask_embed.weight"] = _randn(gen, 1, C, std=0.5)
    sd["mask_embed.conv1.weight"] = _randn(gen, mc // 4, 1, 2, 2, std=0.5)
    sd["mask_embed.conv1.bias"] = _randn(gen, mc // 4, std=0.1)
    _norm(sd, gen, "mask_embed.layer_norm1", mc // 4)
    sd["mask_embed.conv2.weight"] = _randn(gen, mc, mc // 4, 2, 2, std=0.25)
    sd["mask_embed.conv2.bias"] = _randn(gen, mc, std=0.1)
    _norm(sd, gen, "mask_embed.layer_norm2", mc)
    sd["mask_embed.conv3.weight"] = _randn(gen, C, mc, 1, 1, std=0.25)
    sd["mask_embed.conv3.bias"] = _randn(gen, C, std=0.1)
    return sd


def positional_embedding_state_dict(arch: SamVisionArch, seed: int = 3) -> dict[str, torch.Tensor]:
    """``shared_image_embedding.positional_embedding`` (2, num_pos_feats) = scale * randn (HF:549-550).

    A scale of 1.0 keeps the synthetic Fourier features smooth enough to be a meaningful
    numerical test (HF's default 384 for ViT-B turns sin/cos of 2*pi*x into noise)."""
    gen = torch.Generator().manual_seed(seed)
    return {"positional_embedding": _randn(gen, 2, arch.num_pos_feats, std=1.0)}


# ================================================================================================
# RSPrompter-anchor heads (reference module tree, M:53-170 + configs/rsprompter/_base_/rsprompter_anchor.py)
# ================================================================================================
def _conv_sd(sd: dict, gen: torch.Generator, prefix: str, cout: int, cin: int, k: int, bias: bool = True,
             gain: float = 1.0) -> None:
    sd[prefix + ".weight"] = _randn(gen, cout, cin, k, k, std=gain / math.sqrt(cin * k * k))
    if bias:
        sd[prefix + ".bias"] = _randn(gen, cout, std=0.05)


def _bn_sd(sd: dict, gen: torch.Generator, prefix: str, c: int) -> None:
    sd[prefix + ".weight"] = 1.0 + _randn(gen, c, std=0.1)
    sd[prefix + ".bias"] = _randn(gen, c, std=0.1)
    sd[prefix + ".running_mean"] = _randn(gen, c, std=0.1)
    sd[prefix + ".running_var"] = 1.0 + _randn(gen, c, std=0.1).abs()
    sd[prefix + ".num_batches_tracked"] = torch.tensor(100, dtype=torch.long)


def feature_aggregator_state_dict(in_channels: int, n_select: int, hidden: int = 32, out: int = 256,
                                  seed: int = 10) -> dict[str, torch.Tensor]:
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    for i in range(n_select):
        _conv_sd(sd, gen, f"downconvs.{i}.0", hidden, in_channels, 1, gain=1.4)
        _bn_sd(sd, gen, f"downconvs.{i}.1", hidden)
        _conv_sd(sd, gen, f"downconvs.{i}.3", hidden, hidden, 3, gain=1.4)
        _bn_sd(sd, gen, f"downconvs.{i}.4", hidden)
        _conv_sd(sd, gen, f"hidden_convs.{i}.0", hidden, hidden, 3, gain=1.0)
        _bn_sd(sd, gen, f"hidden_convs.{i}.1", hidden)
    _conv_sd(sd, gen, "fusion_conv.0", out, hidden, 1, gain=1.4)
    _bn_sd(sd, gen, "fusion_conv.1", out)
    _conv_sd(sd, gen, "fusion_conv.3", out, out, 3, gain=1.4)
    _bn_sd(sd, gen, "fusion_conv.4", out)
    _conv_sd(sd, gen, "fusion_conv.6", out, out, 3)
    return sd


def pseudo_aggregator_state_dict(in_channels: int = 256, hidden: int = 512, out: int = 256, seed: int = 11):
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    _conv_sd(sd, gen, "channel_fusion.0", hidden, in_channels, 1, bias=False)
    _norm(sd, gen, "channel_fusion.1", hidden)
    _conv_sd(sd, gen, "channel_fusion.2", hidden, hidden, 3, bias=False)
    _norm(sd, gen, "channel_fusion.3", hidden)
    _conv_sd(sd, gen, "channel_fusion.4", out, hidden, 3, bias=False)
    _norm(sd, gen, "channel_fusion.5", out)
    return sd


def simple_fpn_state_dict(bc: int = 256, in_channels=(64, 128, 256, 256), out: int = 256, seed: int = 12):
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}

    def convT(prefix, cin, cout):
        sd[prefix + ".weight"] = _randn(gen, cin, cout, 2, 2, std=1.0 / math.sqrt(cin))
        sd[prefix + ".bias"] = _randn(gen, cout, std=0.05)

    convT("fpn1.0", bc, bc // 2)
    _norm(sd, gen, "fpn1.1", bc // 2)
    convT("fpn1.3", bc // 2, bc // 4)
    convT("fpn2.0", bc, bc // 2)
    for i, c in enumerate(in_channels):
        _conv_sd(sd, gen, f"lateral_convs.{i}.conv", out, c, 1, bias=False)
        _norm(sd, gen, f"lateral_convs.{i}.ln", out)
        _conv_sd(sd, gen, f"fpn_convs.{i}.conv", out, out, 3, bias=False)
        _norm(sd, gen, f"fpn_convs.{i}.ln", out)
    return sd


def rpn_head_state_dict(c: int = 256, num_anchors: int = 6, seed: int = 13):
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    _conv_sd(sd, gen, "rpn_conv", c, c, 3, gain=1.4)
    _conv_sd(sd, gen, "rpn_cls", num_anchors, c, 1, gain=0.3)
    _conv_sd(sd, gen, "rpn_reg", num_anchors * 4, c, 1, gain=0.5)
    return sd


def bbox_head_state_dict(num_classes: int, c: int = 256, roi: int = 7, fc: int = 1024, seed: int = 14):
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    _linear(sd, gen, "shared_fcs.0", fc, c * roi * roi, std=1.4 / math.sqrt(c * roi * roi))
    _linear(sd, gen, "shared_fcs.1", fc, fc, std=1.4 / math.sqrt(fc))
    _linear(sd, gen, "fc_cls", num_classes + 1, fc, std=3.0 / math.sqrt(fc))
    _linear(sd, gen, "fc_reg", 4 * num_classes, fc, std=1.0 / math.sqrt(fc))
    return sd


def mask_head_state_dict(c: int = 256, roi: int = 14, points: int = 5, seed: int = 15):
    """point_emb.* of RSPrompterAnchorMaskHead (M:1641-1651); decoder / no_mask_embed come from the SAM dicts."""
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    _conv_sd(sd, gen, "point_emb.0", c, c, 3, gain=1.4)
    _bn_sd(sd, gen, "point_emb.1", c)
    _linear(sd, gen, "point_emb.4", c, c * roi * roi // 4, std=1.4 / math.sqrt(c * roi * roi // 4))
    _linear(sd, gen, "point_emb.6", c, c, std=1.4 / math.sqrt(c))
    _linear(sd, gen, "point_emb.8", c * 2 * points, c, std=1.0 / math.sqrt(c))
    return sd


def _prefixed(prefix: str, sd: dict) -> dict:
    return {prefix + k: v for k, v in sd.items()}


def anchor_detector_state_dict(arch: SamVisionArch, num_classes: int, n_select: int, seed: int = 0,
                               pseudo_neck: bool = False) -> dict[str, torch.Tensor]:
    """Full RSPrompterAnchor state dict with the reference's key names."""
    sd: dict[str, torch.Tensor] = {}
    sd.update(_prefixed("backbone.vision_encoder.", vision_encoder_state_dict(arch, seed)))
    if pseudo_neck:
        sd.update(_prefixed("neck.feature_aggregator.", pseudo_aggregator_state_dict(seed=seed + 11)))
    else:
        sd.update(_prefixed("neck.feature_aggregator.",
                            feature_aggregator_state_dict(arch.hidden_size, n_select, seed=seed + 10)))
    sd.update(_prefixed("neck.feature_spliter.", simple_fpn_state_dict(seed=seed + 12)))
    sd.update(_prefixed("rpn_head.", rpn_head_state_dict(seed=seed + 13)))
    sd.update(_prefixed("roi_head.bbox_head.", bbox_head_state_dict(num_classes, seed=seed + 14)))
    sd.update(_prefixed("roi_head.mask_head.", mask_head_state_dict(seed=seed + 15)))
    sd.update(_prefixed("roi_head.mask_head.mask_decoder.mask_decoder.", mask_decoder_state_dict(seed=seed + 1)))
    sd["roi_head.mask_head.no_mask_embed.weight"] = prompt_encoder_state_dict(seed=seed + 2)["no_mask_embed.weight"]
    sd.update(_prefixed("shared_image_embedding.shared_image_embedding.",
                        positional_embedding_state_dict(arch, seed + 3)))
    return sd


def fcn_mask_head_state_dict(num_classes: int, c: int = 256, num_convs: int = 4, seed: int = 16):
    """FCNMaskHead (fcn_mask_head.py:68-126): convs.{i}.conv, upsample (ConvTranspose2d), conv_logits."""
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    for i in range(num_convs):
        _conv_sd(sd, gen, f"convs.{i}.conv", c, c, 3, gain=1.4)
    sd["upsample.weight"] = _randn(gen, c, c, 2, 2, std=1.4 / math.sqrt(c))
    sd["upsample.bias"] = _randn(gen, c, std=0.05)
    _conv_sd(sd, gen, "conv_logits", num_classes, c, 1, gain=4.0)
    return sd


def maskrcnn_detector_state_dict(arch: SamVisionArch, num_classes: int, n_select: int, seed: int = 0) -> dict:
    """Full SAMSegMaskRCNN state dict with the reference's key names (M:1218-1244 + _base_/samseg-maskrcnn.py)."""
    sd: dict[str, torch.Tensor] = {}
    sd.update(_prefixed("backbone.vision_encoder.", vision_encoder_state_dict(arch, seed)))
    sd.update(_prefixed("neck.feature_aggregator.",
                        feature_aggregator_state_dict(arch.hidden_size, n_select, seed=seed + 10)))
    sd.update(_prefixed("neck.feature_spliter.", simple_fpn_state_dict(seed=seed + 12)))
    sd.update(_prefixed("rpn_head.", rpn_head_state_dict(num_anchors=3, seed=seed + 13)))
    sd.update(_prefixed("roi_head.bbox_head.", bbox_head_state_dict(num_classes, seed=seed + 14)))
    sd.update(_prefixed("roi_head.mask_head.", fcn_mask_head_state_dict(num_classes, seed=seed + 16)))
    return sd


# ================================================================================================
# RSPrompter-query head (reference module tree, M:274-330 + configs/rsprompter/_base_/rsprompter_query.py)
# ================================================================================================
def _gn_conv_sd(sd: dict, gen: torch.Generator, prefix: str, cout: int, cin: int, k: int, bias: bool) -> None:
    _conv_sd(sd, gen, prefix + ".conv", cout, cin, k, bias=bias, gain=1.2)
    _norm(sd, gen, prefix + ".gn", cout)


def _ffn_sd(sd: dict, gen: torch.Generator, prefix: str, E: int, F: int) -> None:
    _linear(sd, gen, prefix + ".layers.0.0", F, E, std=1.2 / math.sqrt(E))
    _linear(sd, gen, prefix + ".layers.1", E, F, std=1.0 / math.sqrt(F))


def query_head_state_dict(num_classes: int, nq: int = 100, points: int = 5, E: int = 128, C: int = 256, F: int = 512,
                          in_levels: int = 5, enc_levels: int = 3, enc_layers: int = 3, enc_points: int = 4,
                          dec_layers: int = 6, heads: int = 8, seed: int = 20) -> dict[str, torch.Tensor]:
    """RSMask2FormerHead parameters except the SAM decoder / sam_mask_embed (added by the caller)."""
    gen = torch.Generator().manual_seed(seed)
    sd: dict[str, torch.Tensor] = {}
    pd = "pixel_decoder."
    for i in range(enc_levels):
        _gn_conv_sd(sd, gen, f"{pd}input_convs.{i}", E, C, 1, True)
    for l in range(enc_layers):
        p = f"{pd}encoder.layers.{l}."
        _linear(sd, gen, p + "self_attn.sampling_offsets", heads * enc_levels * enc_points * 2, E, std=0.3 / math.sqrt(E))
        sd[p + "self_attn.sampling_offsets.bias"] = _randn(gen, heads * enc_levels * enc_points * 2, std=1.5)
        _linear(sd, gen, p + "self_attn.attention_weights", heads * enc_levels * enc_points, E, std=1.0 / math.sqrt(E))
        _linear(sd, gen, p + "self_attn.value_proj", E, E)
        _linear(sd, gen, p + "self_attn.output_proj", E, E)
        _ffn_sd(sd, gen, p + "ffn", E, F)
        _norm(sd, gen, p + "norms.0", E)
        _norm(sd, gen, p + "norms.1", E)
    sd[pd + "level_encoding.weight"] = _randn(gen, enc_levels, E, std=0.5)
    for i in range(in_levels - enc_levels):
        _gn_conv_sd(sd, gen, f"{pd}lateral_convs.{i}", E, C, 1, False)
        _gn_conv_sd(sd, gen, f"{pd}output_convs.{i}", E, E, 3, False)
    _conv_sd(sd, gen, pd + "mask_feature", C, E, 1, gain=0.5)
    for i in range(dec_layers):
        p = f"transformer_decoder.layers.{i}."
        for a in ("cross_attn", "self_attn"):
            sd[f"{p}{a}.attn.in_proj_weight"] = _randn(gen, 3 * E, E, std=1.3 / math.sqrt(E))
            sd[f"{p}{a}.attn.in_proj_bias"] = _randn(gen, 3 * E, std=0.02)
            _linear(sd, gen, f"{p}{a}.attn.out_proj", E, E)
        _ffn_sd(sd, gen, p + "ffn", E, F)
        for n in range(3):
            _norm(sd, gen, f"{p}norms.{n}", E)
    _norm(sd, gen, "transformer_decoder.post_norm", E)
    sd["query_embed.weight"] = _randn(gen, nq, E, std=1.0)
    sd["query_feat.weight"] = _randn(gen, nq, E, std=1.0)
    sd["level_embed.weight"] = _randn(gen, enc_levels, E, std=0.5)
    _linear(sd, gen, "cls_embed.0", E, E, std=1.4 / math.sqrt(E))
    _linear(sd, gen, "cls_embed.2", num_classes + 1, E, std=2.0 / math.sqrt(E))
    _linear(sd, gen, "mask_embed.0", E, E, std=1.4 / math.sqrt(E))
    _linear(sd, gen, "mask_embed.2", E, E, std=1.4 / math.sqrt(E))
    _linear(sd, gen, "mask_embed.4", C, E, std=1.0 / math.sqrt(E))
    _linear(sd, gen, "point_emb.0", E // 2, E, std=1.4 / math.sqrt(E))
    _linear(sd, gen, "point_emb.2", E // 2, E // 2, std=1.4 / math.sqrt(E // 2))
    _linear(sd, gen, "point_emb.4", C * 2 * points, E // 2, std=1.0 / math.sqrt(E // 2))
    return sd


def query_detector_state_dict(arch: SamVisionArch, num_classes: int, n_select: int, nq: int = 100, points: int = 5,
                              seed: int = 0, pseudo_neck: bool = False) -> dict[str, torch.Tensor]:
    """Full RSPrompterQuery state dict with the reference's key names."""
    sd: dict[str, torch.Tensor] = {}
    sd.update(_prefixed("backbone.vision_encoder.", vision_encoder_state_dict(arch, seed)))
    if pseudo_neck:
        sd.update(_prefixed("neck.feature_aggregator.", pseudo_aggregator_state_dict(seed=seed + 11)))
    else:
        sd.update(_prefixed("neck.feature_aggregator.",
                            feature_aggregator_state_dict(arch.hidden_size, n_select, seed=seed + 10)))
    sd.update(_prefixed("neck.feature_spliter.", simple_fpn_state_dict(seed=seed + 12)))
    sd.update(_prefixed("panoptic_head.", query_head_state_dict(num_classes, nq, points, seed=seed + 20)))
    sd.update(_prefixed("panoptic_head.mask_decoder.mask_decoder.", mask_decoder_state_dict(seed=seed + 1)))
    pe = prompt_encoder_state_dict(seed=seed + 2)
    sd.update({"panoptic_head.sam_" + k: v for k, v in pe.items() if k.startswith("mask_embed.")})
    sd.update(_prefixed("shared_image_embedding.shared_image_embedding.",
                        positional_embedding_state_dict(arch, seed + 3)))
    return sd


def mask2former_head_state_dict(num_classes: int, nq: int = 100, E: int = 256, C: int = 256, F_enc: int = 1024,
                                F_dec: int = 2048, in_levels: int = 5, enc_levels: int = 3, enc_layers: int = 3,
                                enc_points: int = 4, dec_layers: int = 9, heads: int = 8, seed: int = 30) -> dict:
    """Stock Mask2FormerHead parameters (dense_heads/mask2former_head.py:100-141; _base_/samseg-mask2former.py:86-140)."""
    sd = query_head_state_dict(num_classes, nq, points=1, E=E, C=C, F=F_enc, in_levels=in_levels, enc_levels=enc_levels,
                               enc_layers=enc_layers, enc_points=enc_points, dec_layers=0, heads=heads, seed=seed)
    for k in [k for k in sd if k.startswith(("cls_embed.", "point_emb."))]:
        del sd[k]
    gen = torch.Generator().manual_seed(seed + 1)
    for i in range(dec_layers):
        p = f"transformer_decoder.layers.{i}."
        for a in ("cross_attn", "self_attn"):
            sd[f"{p}{a}.attn.in_proj_weight"] = _randn(gen, 3 * E, E, std=1.3 / math.sqrt(E))
            sd[f"{p}{a}.attn.in_proj_bias"] = _randn(gen, 3 * E, std=0.02)
            _linear(sd, gen, f"{p}{a}.attn.out_proj", E, E)
        _ffn_sd(sd, gen, p + "ffn", E, F_dec)
        for n in range(3):
            _norm(sd, gen, f"{p}norms.{n}", E)
    _linear(sd, gen, "cls_embed", num_classes + 1, E, std=2.0 / math.sqrt(E))
    return sd


def mask2former_detector_state_dict(arch: SamVisionArch, num_classes: int, n_select: int, nq: int = 100, seed: int = 0) -> dict:
    """Full SAMSegMask2Former state dict with the reference's key names (M:1247-1274)."""
    sd: dict[str, torch.Tensor] = {}
    sd.update(_prefixed("backbone.vision_encoder.", vision_encoder_state_dict(arch, seed)))
    sd.update(_prefixed("neck.feature_aggregator.",
                        feature_aggregator_state_dict(arch.hidden_size, n_select, seed=seed + 10)))
    sd.update(_prefixed("neck.feature_spliter.", simple_fpn_state_dict(seed=seed + 12)))
    sd.update(_prefixed("panoptic_head.", mask2former_head_state_dict(num_classes, nq, seed=seed + 30)))
    return sd
