"""SAM ViT image encoder on the H100 kernels.

Registry types (M:762-878): ``RSSamVisionEncoder`` (HF ``SamVisionEncoder`` semantics,
HF:1020-1072) and ``MMPretrainSamVisionEncoder`` (``mmpretrain.ViTSAM`` semantics, VS:317-602).
Both keep the reference's parameter names, so HF ``pytorch_model.bin`` checkpoints (prefixes
``module.`` / ``vision_encoder.`` stripped, M:783; mmpretrain renames M:840-851) load unchanged.

Data flow per layer (HF:954-972), all on the C-ABI kernels of ``_lib``:
    LN1 (+ window_partition gather, zero rows for the 64->70 padding)      rsp_layernorm
    qkv Linear                                                             rsp_gemm_bf16
    attention core with in-kernel decomposed rel-pos                       rsp_vit_attention
    proj Linear + window_unpartition scatter + residual add                rsp_gemm_bf16
    LN2                                                                    rsp_layernorm
    lin1 + GELU                                                            rsp_gemm_bf16
    lin2 + residual add  (-> hidden_states[i+1], fp32 NHWC)                rsp_gemm_bf16
The residual stream and LN statistics are fp32; GEMM / attention operands are bf16.
"""
from __future__ import annotations

import re
from collections import OrderedDict

import torch
from torch import nn

from . import _lib
from .registry import MODELS, BaseModule
from .sam_config import SamVisionArch, parse_arch_name, vision_arch

try:  # isinstance(_, SamVisionEncoderOutput) is how the detectors unpack the result (M:99)
    from transformers.models.sam.modeling_sam import SamVisionEncoderOutput as _HFOut
except Exception:  # noqa: BLE001
    _HFOut = None


if _HFOut is not None:
    SamVisionEncoderOutput = _HFOut
else:  # pragma: no cover
    class SamVisionEncoderOutput(tuple):  # type: ignore[no-redef]
        """(last_hidden_state, hidden_states) with attribute access."""

        def __new__(cls, last_hidden_state=None, hidden_states=None, **_):
            items = tuple(x for x in (last_hidden_state, hidden_states) if x is not None)
            self = super().__new__(cls, items)
            self.last_hidden_state = last_hidden_state
            self.hidden_states = hidden_states
            return self


class _Affine(nn.Module):
    """Parameter holder named like nn.Linear / nn.LayerNorm / nn.Conv2d (never called)."""

    def __init__(self, w_shape: tuple[int, ...], bias: bool = True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(w_shape), requires_grad=False)
        if bias:
            self.bias = nn.Parameter(torch.empty(w_shape[0]), requires_grad=False)
        else:
            self.register_parameter("bias", None)


class _Attn(nn.Module):
    def __init__(self, D: int, hd: int, S: int):
        super().__init__()
        self.rel_pos_h = nn.Parameter(torch.empty(2 * S - 1, hd), requires_grad=False)
        self.rel_pos_w = nn.Parameter(torch.empty(2 * S - 1, hd), requires_grad=False)
        self.qkv = _Affine((3 * D, D))
        self.proj = _Affine((D, D))


class _Mlp(nn.Module):
    def __init__(self, D: int, M: int):
        super().__init__()
        self.lin1 = _Affine((M, D))
        self.lin2 = _Affine((D, M))


class _Layer(nn.Module):
    def __init__(self, arch: SamVisionArch, S: int):
        super().__init__()
        D = arch.hidden_size
        self.layer_norm1 = _Affine((D,))
        self.attn = _Attn(D, arch.head_dim, S)
        self.layer_norm2 = _Affine((D,))
        self.mlp = _Mlp(D, arch.mlp_dim)


class _PatchEmbed(nn.Module):
    def __init__(self, D: int, p: int):
        super().__init__()
        self.projection = _Affine((D, 3, p, p))


class _Neck(nn.Module):
    def __init__(self, D: int, C: int):
        super().__init__()
        self.conv1 = _Affine((C, D, 1, 1), bias=False)
        self.layer_norm1 = _Affine((C,))
        self.conv2 = _Affine((C, C, 3, 3), bias=False)
        self.layer_norm2 = _Affine((C,))


def window_maps(batch: int, grid: int, window: int, device: torch.device) -> tuple[torch.Tensor, int]:
    """int32 [B * nW * nW * window^2]: token row of every windowed row, -1 for padding.

    One array serves both directions: as the LN1 gather map (window_partition, HF:900-922) and
    as the proj-GEMM scatter map (window_unpartition + crop, HF:925-952)."""
    nw = (grid + window - 1) // window
    gp = nw * window
    ys = torch.arange(gp, device=device)
    tok = ys[:, None] * grid + ys[None, :]
    tok = torch.where((ys[:, None] < grid) & (ys[None, :] < grid), tok, torch.full_like(tok, -1))
    tok = tok.reshape(nw, window, nw, window).permute(0, 2, 1, 3).reshape(-1)  # (wy, wx, iy, ix)
    off = (torch.arange(batch, device=device) * grid * grid)[:, None]
    full = torch.where(tok[None, :] >= 0, tok[None, :] + off, torch.full_like(tok[None, :], -1))
    return full.reshape(-1).to(torch.int32).contiguous(), nw * nw


class SamVisionEncoderB200(nn.Module):
    """HF ``SamVisionEncoder`` parameter tree with a forward made of H100 kernels."""

    def __init__(self, arch: SamVisionArch):
        super().__init__()
        self.arch = arch
        D, g = arch.hidden_size, arch.grid
        self.patch_embed = _PatchEmbed(D, arch.patch_size)
        self.pos_embed = nn.Parameter(torch.empty(1, g, g, D), requires_grad=False)
        self.layers = nn.ModuleList(
            _Layer(arch, g if i in arch.global_attn_indexes else arch.window_size)
            for i in range(arch.num_layers))
        self.neck = _Neck(D, arch.output_channels)
        self._prep: dict | None = None
        self._maps: dict = {}
        self.register_load_state_dict_post_hook(lambda *_: self._invalidate())
        self._register_load_state_dict_pre_hook(self._resize_checkpoint_tables)

    def _resize_checkpoint_tables(self, state_dict, prefix, *args):
        """A checkpoint trained at another image size (a 1024^2 SAM checkpoint into the 512^2 model of the *-peft-512
        configs): absolute position embedding resized bicubically, relative-position tables linearly, exactly as
        mmpretrain ViTSAM does at load time (VS:611-662, mmpretrain/models/utils/embed.py:16-59)."""
        import torch.nn.functional as F
        k = prefix + "pos_embed"
        if k in state_dict and tuple(state_dict[k].shape) != tuple(self.pos_embed.shape):
            src = state_dict[k]
            dst = F.interpolate(src.permute(0, 3, 1, 2).float(), size=tuple(self.pos_embed.shape[1:3]), mode="bicubic",
                                align_corners=False)
            state_dict[k] = dst.permute(0, 2, 3, 1).to(src.dtype).contiguous()
        for name, own in self.named_parameters():
            if "rel_pos_" not in name:
                continue
            ck = prefix + name
            if ck in state_dict and state_dict[ck].shape[0] != own.shape[0]:
                t = state_dict[ck]
                L1, L2 = t.shape[0], own.shape[0]
                new = F.interpolate(t.reshape(1, L1, -1).permute(0, 2, 1), size=L2, mode="linear")
                state_dict[ck] = new.reshape(-1, L2).permute(1, 0).contiguous()

    def _invalidate(self) -> None:
        self._prep = None

    def _apply(self, fn, *a, **k):  # .to() / .cuda() change storage: rebuild kernel weights
        self._prep = None
        return super()._apply(fn, *a, **k)

    # ---------------------------------------------------------------- kernel-side weights
    @torch.no_grad()
    def _prepare(self) -> dict:
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise _lib.RspError("SamVisionEncoderB200 runs on CUDA only; move the module to a H100")
        bf = lambda t: t.detach().to(dtype=torch.bfloat16).contiguous()  # noqa: E731
        f32 = lambda t: t.detach().to(dtype=torch.float32).contiguous()  # noqa: E731
        a = self.arch
        D, C = a.hidden_size, a.output_channels
        p: dict = {}
        p["pe_w"] = bf(self.patch_embed.projection.weight.reshape(D, -1))
        p["pe_b"] = f32(self.patch_embed.projection.bias)
        p["pos"] = f32(self.pos_embed.reshape(-1, D))
        layers = []
        for lyr in self.layers:
            layers.append(dict(
                ln1_w=f32(lyr.layer_norm1.weight), ln1_b=f32(lyr.layer_norm1.bias),
                ln2_w=f32(lyr.layer_norm2.weight), ln2_b=f32(lyr.layer_norm2.bias),
                qkv_w=bf(lyr.attn.qkv.weight), qkv_b=f32(lyr.attn.qkv.bias),
                proj_w=bf(lyr.attn.proj.weight), proj_b=f32(lyr.attn.proj.bias),
                rel_h=bf(lyr.attn.rel_pos_h), rel_w=bf(lyr.attn.rel_pos_w),
                lin1_w=bf(lyr.mlp.lin1.weight), lin1_b=f32(lyr.mlp.lin1.bias),
                lin2_w=bf(lyr.mlp.lin2.weight), lin2_b=f32(lyr.mlp.lin2.bias)))
        p["layers"] = layers
        p["n1_w"] = bf(self.neck.conv1.weight.reshape(C, D))
        p["n2_w"] = bf(self.neck.conv2.weight.permute(0, 2, 3, 1).reshape(C, 9 * C))
        p["nln1_w"], p["nln1_b"] = f32(self.neck.layer_norm1.weight), f32(self.neck.layer_norm1.bias)
        p["nln2_w"], p["nln2_b"] = f32(self.neck.layer_norm2.weight), f32(self.neck.layer_norm2.bias)
        self._prep = p
        return p

    def _window_map(self, batch: int, device: torch.device) -> tuple[torch.Tensor, int]:
        key = (batch, device)
        if key not in self._maps:
            self._maps[key] = window_maps(batch, self.arch.grid, self.arch.window_size, device)
        return self._maps[key]

    # ---------------------------------------------------------------- forward
    @torch.no_grad()
    def encode(self, pixel_values: torch.Tensor, want_hidden: bool = True, bf16_copies: dict | None = None):
        """Returns (embeddings fp32 [B,C,g,g], [hidden_states fp32 [B,g,g,D]] * (L+1), embeddings NHWC).
        bf16_copies: dict whose keys are hidden-state indices i < L; on return bf16_copies[i] is a bf16 [B,g,g,D] copy
        of hidden_states[i], written by layer i's LN1 kernel while it reads that state (no separate cast pass)."""
        a = self.arch
        if pixel_values.dim() != 4 or pixel_values.shape[1] != 3:
            raise ValueError("Make sure that the channel dimension of the pixel values match with the "
                             "one set in the configuration.")
        B, _, Hi, Wi = pixel_values.shape
        if Hi != a.image_size or Wi != a.image_size:
            raise ValueError(f"Input image size ({Hi}*{Wi}) doesn't match model ({a.image_size}*{a.image_size}).")
        p = self._prep or self._prepare()
        D, g, H, hd, C = a.hidden_size, a.grid, a.num_heads, a.head_dim, a.output_channels
        T = g * g
        M = B * T
        if pixel_values.dtype == torch.uint8:
            # DetDataPreprocessor fused into the operand loader: raw uint8 pixels (NCHW or channels-last memory) ->
            # normalised bf16 patch rows; (mean, std, swap_rb) ride on the tensor (preprocess.py)
            norm = getattr(pixel_values, "rsp_norm", None)
            if norm is None:
                raise _lib.RspError("uint8 pixel_values need the DetDataPreprocessor normalisation (tensor.rsp_norm)")
            x = pixel_values
            patches = _lib.patchify16_u8(x, norm[0], norm[1], norm[2])
        else:
            x = pixel_values.to(dtype=torch.float32).contiguous()
            patches = _lib.patchify16(x)
        h = _lib.gemm(patches, p["pe_w"], p["pe_b"], residual=p["pos"], res_mod=T,
                      out_dtype=torch.float32)
        hidden = [h]
        wmap, n_win = self._window_map(B, x.device)
        ws = a.window_size
        for i, lw in enumerate(p["layers"]):
            is_global = i in a.global_attn_indexes
            cp = None
            if bf16_copies is not None and i in bf16_copies:
                cp = torch.empty(M, D, device=x.device, dtype=torch.bfloat16)
                bf16_copies[i] = cp.view(B, g, g, D)
            if is_global:
                xn = _lib.layernorm(h, lw["ln1_w"], lw["ln1_b"], a.layer_norm_eps, copy_out=cp)
                qkv = _lib.gemm(xn, lw["qkv_w"], lw["qkv_b"])
                att = _lib.vit_attention(qkv, lw["rel_h"], lw["rel_w"], B, g, H, hd)
                x1 = _lib.gemm(att, lw["proj_w"], lw["proj_b"], residual=h, out_dtype=torch.float32)
            else:
                xn = _lib.layernorm(h, lw["ln1_w"], lw["ln1_b"], a.layer_norm_eps, src_map=wmap, copy_out=cp)
                qkv = _lib.gemm(xn, lw["qkv_w"], lw["qkv_b"])
                # window_unpartition + crop happen in the attention store: the projection is a plain GEMM
                att = _lib.vit_attention(qkv, lw["rel_h"], lw["rel_w"], B * n_win, ws, H, hd, out_row_map=wmap,
                                         out_rows=M)
                x1 = _lib.gemm(att, lw["proj_w"], lw["proj_b"], residual=h, out_dtype=torch.float32)
            xn2 = _lib.layernorm(x1, lw["ln2_w"], lw["ln2_b"], a.layer_norm_eps)
            y = _lib.gemm(xn2, lw["lin1_w"], lw["lin1_b"], act="gelu")
            h = _lib.gemm(y, lw["lin2_w"], lw["lin2_b"], residual=x1, out_dtype=torch.float32)
            hidden.append(h)
        # neck: 1x1 conv -> LN over C -> 3x3 conv -> LN over C (HF:975-992), channels-last
        hb = _lib.cast_bf16(h)
        c1 = _lib.gemm(hb, p["n1_w"])
        l1 = _lib.layernorm(c1, p["nln1_w"], p["nln1_b"], 1e-6)
        if _lib.conv3x3_ok(B, g, g, C):
            c2 = _lib.conv3x3_nhwc(l1.view(B, g, g, C), p["n2_w"])
        else:
            c2 = _lib.gemm(_lib.im2col_nhwc(l1.view(B, g, g, C), 3, 3, 1, 1), p["n2_w"])
        l2 = _lib.layernorm(c2, p["nln2_w"], p["nln2_b"], 1e-6, out_dtype=torch.float32)
        emb = _lib.nhwc_to_nchw(l2.view(B, g, g, C))
        hs = tuple(t.view(B, g, g, D) for t in hidden) if want_hidden else None
        return emb, hs, l2.view(B, g, g, C)

    def forward(self, pixel_values: torch.Tensor | None = None, **kwargs):
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        emb, hs, _ = self.encode(pixel_values, want_hidden=self.arch.output_hidden_states)
        return SamVisionEncoderOutput(last_hidden_state=emb, hidden_states=hs)


def strip_checkpoint_prefixes(state_dict: dict, revise_keys=((r"^module\.", ""), (r"^vision_encoder\.", ""))):
    """mmengine load_checkpoint(revise_keys=...) semantics (M:777-783)."""
    out = OrderedDict()
    for k, v in state_dict.items():
        for pat, rep in revise_keys:
            k = re.sub(pat, rep, k)
        out[k] = v
    return out


def merge_lora_into_qkv(state_dict: dict, r_alpha: tuple[int, int] = (16, 32)) -> dict:
    """Fold peft LoRA factors into qkv.weight: W += (alpha / r) * B @ A (M:785-797)."""
    r, alpha = r_alpha
    out = OrderedDict()
    for k, v in state_dict.items():
        k2 = k.replace("base_model.model.", "").replace(".base_layer.", ".")
        if "lora_A" in k2 or "lora_B" in k2:
            continue
        out[k2] = v
    for k, v in state_dict.items():
        if "lora_A" in k:
            base = k.replace("base_model.model.", "").split(".lora_A")[0]
            bk = k.replace("lora_A", "lora_B")
            if bk in state_dict and base + ".weight" in out:
                out[base + ".weight"] = out[base + ".weight"] + (alpha / r) * (state_dict[bk] @ v)
    return out


def _install_lora_merge_hook(wrapper: nn.Module, peft_config: dict | None) -> None:
    """Checkpoints of the reference's peft-wrapped encoder (M:785-797: keys ``vision_encoder.base_model.model.*``,
    ``qkv.base_layer.weight``, ``qkv.lora_A/B.default.weight``) load into the plain module with the LoRA update
    folded into qkv.weight - inference needs no adapter branch."""
    cfg = dict(r=16, lora_alpha=32)
    cfg.update(peft_config or {})
    r_alpha = (int(cfg["r"]), int(cfg["lora_alpha"]))

    def hook(state_dict, prefix, *args):
        pre = prefix + "vision_encoder."
        keys = [k for k in state_dict if k.startswith(pre)]
        if not any("lora_" in k or ".base_layer." in k or "base_model.model." in k for k in keys):
            return
        sub = OrderedDict((k[len(pre):], state_dict.pop(k)) for k in keys)
        for k, v in merge_lora_into_qkv(sub, r_alpha).items():
            state_dict[pre + k] = v

    wrapper._register_load_state_dict_pre_hook(hook)


def _load_pretrained(module: nn.Module, init_cfg: dict | None, revise_keys) -> None:
    if not init_cfg or not init_cfg.get("checkpoint"):
        return
    import os
    path = os.path.expanduser(init_cfg["checkpoint"])
    if not os.path.isfile(path):
        raise FileNotFoundError(f"init_cfg checkpoint {path} not found")
    if path.endswith(".safetensors"):           # HF hub snapshots ship model.safetensors next to pytorch_model.bin
        from safetensors.torch import load_file
        sd = load_file(path, device="cpu")
    else:
        sd = torch.load(path, map_location="cpu")
    sd = sd.get("state_dict", sd)
    sd = strip_checkpoint_prefixes(sd, revise_keys)
    own = module.state_dict()
    module.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)


@MODELS.register_module(force=True)
class RSSamVisionEncoder(BaseModule):
    """Drop-in for mmdet.rsprompter RSSamVisionEncoder (M:762-809)."""

    def __init__(self, hf_pretrain_name, extra_config=None, peft_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        arch = vision_arch(hf_pretrain_name, extra_config)
        self.vision_encoder = SamVisionEncoderB200(arch)
        self.peft_config = peft_config  # LoRA is merged at load time for inference
        _install_lora_merge_hook(self, peft_config)
        _load_pretrained(self.vision_encoder, init_cfg, [(r"^module\.", ""), (r"^vision_encoder\.", "")])
        self.vision_encoder.is_init = True

    def init_weights(self):
        pass

    def forward(self, *args, **kwargs):
        return self.vision_encoder(*args, **kwargs)


# mmpretrain ViTSAM parameter names -> HF names (inverse of the revise_keys at M:840-851)
_MMPRETRAIN_TO_HF = [
    (r"\.ln1\.", ".layer_norm1."), (r"\.ln2\.", ".layer_norm2."),
    (r"\.ffn\.layers\.0\.0\.", ".mlp.lin1."), (r"\.ffn\.layers\.1\.", ".mlp.lin2."),
    (r"^channel_reduction\.0\.", "neck.conv1."), (r"^channel_reduction\.1\.", "neck.layer_norm1."),
    (r"^channel_reduction\.2\.", "neck.conv2."), (r"^channel_reduction\.3\.", "neck.layer_norm2."),
]


@MODELS.register_module(force=True)
class MMPretrainSamVisionEncoder(BaseModule):
    """Drop-in for MMPretrainSamVisionEncoder (M:812-878): any img_size, 1-tuple output.

    ``mmpretrain.ViTSAM`` (VS:570-602) with ``out_indices=[-1]`` returns only the neck output;
    the absolute position embedding is stored at ``img_size`` resolution and the relative
    tables at 2*size-1 (resized at checkpoint load, VS:636-662)."""

    def __init__(self, hf_pretrain_name, img_size=1024, peft_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        name = hf_pretrain_name.split("-")[-1].split("_")[-1]
        arch = vision_arch(name if name in ("base", "large", "huge") else hf_pretrain_name,
                           img_size=img_size)
        self.vision_encoder = SamVisionEncoderB200(arch)
        self.peft_config = peft_config
        _install_lora_merge_hook(self, peft_config)
        self._register_load_state_dict_pre_hook(self._rename_mmpretrain_keys)
        _load_pretrained(self.vision_encoder, init_cfg, [(r"^module\.", ""), (r"^vision_encoder\.", "")])
        self.vision_encoder.is_init = True

    def init_weights(self):
        pass

    @staticmethod
    def _rename_mmpretrain_keys(state_dict, prefix, *args):
        """A checkpoint saved from the reference module carries mmpretrain ViTSAM parameter names (ln1, ffn.layers,
        channel_reduction: the forward direction of the revise_keys at M:840-851); map them onto this module's."""
        pre = prefix + "vision_encoder."
        for k in [k for k in state_dict if k.startswith(pre)]:
            k2 = k[len(pre):]
            for pat, rep in _MMPRETRAIN_TO_HF:
                k2 = re.sub(pat, rep, k2)
            if pre + k2 != k:
                state_dict[pre + k2] = state_dict.pop(k)

    def load_mmpretrain_state_dict(self, sd: dict) -> None:
        out = OrderedDict()
        for k, v in sd.items():
            for pat, rep in _MMPRETRAIN_TO_HF:
                k = re.sub(pat, rep, k)
            out[k] = v
        self.vision_encoder.load_state_dict(out)

    def forward(self, x):
        emb, _, _ = self.vision_encoder.encode(x, want_hidden=False)
        return (emb,)


__all__ = ["SamVisionEncoderB200", "RSSamVisionEncoder", "MMPretrainSamVisionEncoder",
           "SamVisionEncoderOutput", "window_maps", "parse_arch_name"]
