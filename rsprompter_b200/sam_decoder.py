"""SAM mask decoder, positional embedding and prompt-encoder members on the H100 kernels.

Registry types (M:744-759, 881-914): ``RSSamMaskDecoder``, ``RSSamPositionalEmbedding``,
``RSSamPromptEncoder``; parameter names are HF's (``mask_decoder.*`` etc.) so
``pytorch_model.bin`` loads unchanged.

Decoder data flow (HF:461-543 over HF:306-405), N prompts, Tt = 5 + P tokens, HW image tokens:
  * every Linear / ConvTranspose is ``rsp_gemm_bf16(_ex)``; the LayerNorm that follows an
    out_proj / lin2 is fused into that GEMM's epilogue (epi_mode 1), so the pre-norm sums never
    reach HBM;
  * ``k_proj(keys + pe) = k_proj(keys) + k_proj(pe)``: the positional half is projected once
    per call on HW rows and added as a broadcast residual in the epilogue;
  * prompts of one image share its embedding through block maps (``res_block_map`` /
    ``kv_block`` / ``q_block``) instead of the ``repeat_interleave`` copies of M:367-368,1682-1683
    (3 x N x 4 MB in the reference);
  * upscaling: conv-transpose 1 + LayerNorm2d + GELU is one GEMM (epi_mode 2), conv-transpose 2
    + GELU + the hypernetwork product is another (epi_mode 3): the (N, 32, 4h, 4w) upscaled
    embedding is never materialised.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from . import _lib
from .registry import MODELS, BaseModule
from .sam_config import SamDecoderArch, decoder_arch, vision_arch
from .sam_encoder import _Affine, _load_pretrained


class _Embedding(nn.Module):
    def __init__(self, n: int, c: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n, c), requires_grad=False)


class _SamAttention(nn.Module):
    def __init__(self, C: int, internal: int):
        super().__init__()
        self.q_proj = _Affine((internal, C))
        self.k_proj = _Affine((internal, C))
        self.v_proj = _Affine((internal, C))
        self.out_proj = _Affine((C, internal))


class _Mlp(nn.Module):
    def __init__(self, C: int, M: int):
        super().__init__()
        self.lin1 = _Affine((M, C))
        self.lin2 = _Affine((C, M))


class _TwoWayBlock(nn.Module):
    def __init__(self, a: SamDecoderArch):
        super().__init__()
        C = a.hidden_size
        self.self_attn = _SamAttention(C, C)
        self.layer_norm1 = _Affine((C,))
        self.cross_attn_token_to_image = _SamAttention(C, C // a.attention_downsample_rate)
        self.layer_norm2 = _Affine((C,))
        self.mlp = _Mlp(C, a.mlp_dim)
        self.layer_norm3 = _Affine((C,))
        self.layer_norm4 = _Affine((C,))
        self.cross_attn_image_to_token = _SamAttention(C, C // a.attention_downsample_rate)


class _TwoWayTransformer(nn.Module):
    def __init__(self, a: SamDecoderArch):
        super().__init__()
        self.layers = nn.ModuleList(_TwoWayBlock(a) for _ in range(a.num_layers))
        self.final_attn_token_to_image = _SamAttention(a.hidden_size, a.hidden_size // a.attention_downsample_rate)
        self.layer_norm_final_attn = _Affine((a.hidden_size,))


class _FeedForward(nn.Module):
    def __init__(self, cin: int, hidden: int, cout: int, num_layers: int):
        super().__init__()
        self.proj_in = _Affine((hidden, cin))
        self.proj_out = _Affine((cout, hidden))
        self.layers = nn.ModuleList(_Affine((hidden, hidden)) for _ in range(num_layers - 2))


class _ConvT(nn.Module):
    def __init__(self, cin: int, cout: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cin, cout, 2, 2), requires_grad=False)
        self.bias = nn.Parameter(torch.empty(cout), requires_grad=False)


class SamMaskDecoderB200(nn.Module):
    """HF ``SamMaskDecoder`` parameter tree; ``decode`` runs on the H100 kernels."""

    def __init__(self, arch: SamDecoderArch | None = None):
        super().__init__()
        a = self.arch = arch or SamDecoderArch()
        C = a.hidden_size
        self.num_mask_tokens = a.num_multimask_outputs + 1
        self.iou_token = _Embedding(1, C)
        self.mask_tokens = _Embedding(self.num_mask_tokens, C)
        self.transformer = _TwoWayTransformer(a)
        self.upscale_conv1 = _ConvT(C, C // 4)
        self.upscale_conv2 = _ConvT(C // 4, C // 8)
        self.upscale_layer_norm = _Affine((C // 4,))
        self.output_hypernetworks_mlps = nn.ModuleList(
            _FeedForward(C, C, C // 8, 3) for _ in range(self.num_mask_tokens))
        self.iou_prediction_head = _FeedForward(C, a.iou_head_hidden_dim, self.num_mask_tokens, a.iou_head_depth)
        self._prep: dict | None = None
        self.register_load_state_dict_post_hook(lambda *_: setattr(self, "_prep", None))

    def _apply(self, fn, *a, **k):
        self._prep = None
        return super()._apply(fn, *a, **k)

    # ------------------------------------------------------------------ kernel-side weights
    @torch.no_grad()
    def _prepare(self) -> dict:
        if self.iou_token.weight.device.type != "cuda":
            raise _lib.RspError("SamMaskDecoderB200 runs on CUDA only")
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()  # noqa: E731
        f32 = lambda t: t.detach().to(torch.float32).contiguous()  # noqa: E731

        def attn(m: _SamAttention) -> dict:
            return dict(qw=bf(m.q_proj.weight), qb=f32(m.q_proj.bias), kw=bf(m.k_proj.weight),
                        kb=f32(m.k_proj.bias), vw=bf(m.v_proj.weight), vb=f32(m.v_proj.bias),
                        ow=bf(m.out_proj.weight), ob=f32(m.out_proj.bias),
                        # k | v of the image tokens as one projection (the keys are read once)
                        kvw=bf(torch.cat([m.k_proj.weight, m.v_proj.weight], dim=0)),
                        kvb=f32(torch.cat([m.k_proj.bias, m.v_proj.bias], dim=0)))

        def ln(m: _Affine) -> tuple:
            return (f32(m.weight), f32(m.bias))

        def ff(m: _FeedForward) -> list:
            mods = [m.proj_in, *m.layers, m.proj_out]
            return [(bf(x.weight), f32(x.bias)) for x in mods]

        p: dict = {"layers": []}
        for blk in self.transformer.layers:
            p["layers"].append(dict(
                sa=attn(blk.self_attn), t2i=attn(blk.cross_attn_token_to_image),
                i2t=attn(blk.cross_attn_image_to_token),
                w1=bf(blk.mlp.lin1.weight), b1=f32(blk.mlp.lin1.bias),
                w2=bf(blk.mlp.lin2.weight), b2=f32(blk.mlp.lin2.bias),
                ln1=ln(blk.layer_norm1), ln2=ln(blk.layer_norm2), ln3=ln(blk.layer_norm3),
                ln4=ln(blk.layer_norm4)))
        p["final"] = attn(self.transformer.final_attn_token_to_image)
        p["lnf"] = ln(self.transformer.layer_norm_final_attn)
        c4, c8 = self.upscale_conv1.weight.shape[1], self.upscale_conv2.weight.shape[1]
        # ConvTranspose2d(k=2, s=2) as a GEMM whose output columns are (tap = ty*2+tx, channel)
        p["up1_w"] = bf(self.upscale_conv1.weight.permute(2, 3, 1, 0).reshape(4 * c4, -1))
        p["up1_b"] = f32(self.upscale_conv1.bias.repeat(4))
        p["up_ln"] = ln(self.upscale_layer_norm)
        p["up2_w"] = bf(self.upscale_conv2.weight.permute(2, 3, 1, 0).reshape(4 * c8, -1))
        p["up2_b"] = f32(self.upscale_conv2.bias.repeat(4))
        p["hyper"] = [ff(m) for m in self.output_hypernetworks_mlps]
        p["iou"] = ff(self.iou_prediction_head)
        p["out_tokens"] = f32(torch.cat([self.iou_token.weight, self.mask_tokens.weight], dim=0))
        p["pos_terms"] = {}
        self._prep = p
        return p

    def _pos_terms(self, p: dict, pos_rows: torch.Tensor) -> dict:
        """"keys + key_point_embedding" (HF:326, 339-340) never exists as a tensor:
        (keys + pos) W^T = keys W^T + pos W^T, and pos W^T (bf16 [HW, n], a constant of the weights and the map
        size) enters the projection as a broadcast residual slab of the GEMM epilogue."""
        key = (pos_rows.data_ptr(), pos_rows.shape[0])
        if key not in p["pos_terms"]:
            pb = _lib.cast_bf16(pos_rows)
            layers = [L["t2i"] for L in p["layers"]] + [p["final"]]
            kv = []
            for a in layers:
                t = torch.zeros(pos_rows.shape[0], a["kvw"].shape[0], device=pos_rows.device, dtype=torch.bfloat16)
                n_k = a["kw"].shape[0]
                t[:, :n_k] = _lib.gemm(pb, a["kw"])                  # v half stays 0
                kv.append(t)
            q = [_lib.gemm(pb, L["i2t"]["qw"]) for L in p["layers"]]
            p["pos_terms"] = {key: dict(kv=kv, q=q)}
        return p["pos_terms"][key]

    @staticmethod
    def _ff(x_bf: torch.Tensor, layers: list) -> torch.Tensor:
        """SamFeedForward (HF:408-429): ReLU after every layer but the last; fp32 result."""
        h = x_bf
        for w, b in layers[:-1]:
            h = _lib.gemm(h, w, b, act="relu")
        w, b = layers[-1]
        return _lib.gemm(h, w, b, out_dtype=torch.float32)

    # ------------------------------------------------------------------ decode
    @torch.no_grad()
    def decode(self, emb_rows: torch.Tensor, pos_rows: torch.Tensor, sparse: torch.Tensor,
               hw: tuple[int, int], prompt_img: torch.Tensor | None = None,
               dense_vec: torch.Tensor | None = None, dense_rows: torch.Tensor | None = None,
               multimask_output: bool = False, src_pair: tuple | None = None):
        """emb_rows fp32 [Bi*HW, C] channels-last image embeddings (Bi images, or N when
        prompt_img is None); pos_rows fp32 [HW, C]; sparse fp32 [N, P, C]; prompt_img int32 [N]
        image of each prompt; dense_vec fp32 [C] (no_mask_embed broadcast, M:1680) or dense_rows
        fp32 [N*HW, C] per-prompt dense embeddings (M:362).
        -> masks fp32 [N, n_out, 4h, 4w], iou fp32 [N, n_out]."""
        p = self._prep or self._prepare()
        a = self.arch
        C, H = a.hidden_size, a.num_heads
        h, w = hw
        HW = h * w
        N, P, _ = sparse.shape
        Tt = 1 + self.num_mask_tokens + P
        dev = sparse.device
        assert pos_rows.shape == (HW, C) and (emb_rows is None or emb_rows.shape[1] == C)
        shared = prompt_img is not None and dense_rows is None
        pos_rows = pos_rows.contiguous()
        # ---- src = image_embeddings + dense (HF:499)
        if src_pair is not None:
            # per-prompt sources already built on the device (rsp_mask_embed_src): bf16 src
            src_b = src_pair[0]
            src32, blk = src_b, None
        elif dense_rows is not None:
            if prompt_img is not None:  # per-prompt dense on per-image embeddings: expand once
                emb_rows = emb_rows.view(-1, HW, C)[prompt_img.long()].reshape(N * HW, C)
            src32 = emb_rows + dense_rows
            blk = None
        else:
            src32 = emb_rows if dense_vec is None else emb_rows + dense_vec.view(1, C)
            blk = prompt_img if shared else None
        if src_pair is None:
            src32 = src32.contiguous()
            src_b = _lib.cast_bf16(src32)
        pt = self._pos_terms(p, pos_rows)
        tokens = torch.cat([p["out_tokens"].unsqueeze(0).expand(N, -1, -1), sparse.to(torch.float32)], dim=1)
        tokens = tokens.reshape(N * Tt, C).contiguous()

        def t2i(layer: dict, queries: torch.Tensor, keys_b: torch.Tensor, pos_kv: torch.Tensor, kv_blk, ln):
            qin = _lib.add_cast_bf16(queries, tokens)
            q = _lib.gemm(qin, layer["qw"], layer["qb"])
            KV = _lib.gemm(keys_b, layer["kvw"], layer["kvb"], residual=pos_kv, res_mod=HW)   # [rows, k | v]
            n_k = layer["kw"].shape[0]
            att = _lib.t2i_attention(q.view(N, Tt, -1), KV[:, :n_k], KV[:, n_k:], HW, kv_block=kv_blk)
            return _lib.gemm(att.view(N * Tt, -1), layer["ow"], layer["ob"], residual=queries,
                             out_dtype=torch.float32, ln=ln)

        keys_b, keys_res, kblk = src_b, src_b, blk
        queries = None
        for li, L in enumerate(p["layers"]):
            sa = L["sa"]
            if li == 0:  # skip_first_layer_pe: attention output replaces the queries (HF:316-317)
                tb = _lib.cast_bf16(tokens)
                q = _lib.gemm(tb, sa["qw"], sa["qb"])
                k = _lib.gemm(tb, sa["kw"], sa["kb"])
                v = _lib.gemm(tb, sa["vw"], sa["vb"])
                att = _lib.token_self_attention(q.view(N, Tt, C), k.view(N, Tt, C), v.view(N, Tt, C), H)
                queries = _lib.gemm(att.view(N * Tt, C), sa["ow"], sa["ob"], out_dtype=torch.float32,
                                    ln=(*L["ln1"], a.layer_norm_eps))
            else:
                qin = _lib.add_cast_bf16(queries, tokens)
                q = _lib.gemm(qin, sa["qw"], sa["qb"])
                k = _lib.gemm(qin, sa["kw"], sa["kb"])
                v = _lib.gemm(_lib.cast_bf16(queries), sa["vw"], sa["vb"])
                att = _lib.token_self_attention(q.view(N, Tt, C), k.view(N, Tt, C), v.view(N, Tt, C), H)
                queries = _lib.gemm(att.view(N * Tt, C), sa["ow"], sa["ob"], residual=queries,
                                    out_dtype=torch.float32, ln=(*L["ln1"], a.layer_norm_eps))
            # tokens -> image cross attention (HF:323-333)
            queries = t2i(L["t2i"], queries, keys_b, pt["kv"][li], kblk, (*L["ln2"], a.layer_norm_eps))
            # MLP (HF:335-338)
            hdn = _lib.gemm(_lib.cast_bf16(queries), L["w1"], L["b1"], act="relu")
            queries = _lib.gemm(hdn, L["w2"], L["b2"], residual=queries, out_dtype=torch.float32,
                                ln=(*L["ln3"], a.layer_norm_eps))
            # image -> tokens cross attention (HF:340-347)
            i2t = L["i2t"]
            qin = _lib.add_cast_bf16(queries, tokens)
            ktok = _lib.gemm(qin, i2t["kw"], i2t["kb"])
            vtok = _lib.gemm(_lib.cast_bf16(queries), i2t["vw"], i2t["vb"])
            Qimg = _lib.gemm(keys_b, i2t["qw"], i2t["qb"], residual=pt["q"][li], res_mod=HW)
            att = _lib.i2t_attention(Qimg, ktok.view(N, Tt, -1), vtok.view(N, Tt, -1), HW, q_block=kblk)
            # keys = LN4(keys + out_proj(attn)) (HF:346-347) in the out_proj GEMM's epilogue: the residual slab
            # (block-mapped prompt -> image in the first layer) arrives by TMA, the row statistics are taken on
            # the fp32 accumulator, and only the normalised bf16 keys are written
            keys_b = _lib.gemm(att, i2t["ow"], i2t["ob"], residual=keys_res, ln=(*L["ln4"], a.layer_norm_eps),
                               res_block_map=kblk, res_block_rows=HW if kblk is not None else 0)
            keys_res, kblk = keys_b, None
        queries = t2i(p["final"], queries, keys_b, pt["kv"][-1], None, (*p["lnf"], 1e-5))
        qv = queries.view(N, Tt, C)
        iou_tok = _lib.cast_bf16(qv[:, 0].contiguous())
        iou = self._ff(iou_tok, p["iou"])                                   # [N, num_mask_tokens]
        # upscaling + hypernetwork product (HF:515-531)
        up1 = _lib.gemm(keys_b, p["up1_w"], p["up1_b"], ln64_gelu=(*p["up_ln"], 1e-6))   # [N*HW, 4*64]
        up1 = up1.view(N * HW * 4, -1)
        sel = range(1, self.num_mask_tokens) if multimask_output else range(0, 1)
        masks = []
        for i in sel:
            mt = _lib.cast_bf16(qv[:, 1 + i].contiguous())
            hyper = self._ff(mt, p["hyper"][i])                             # [N, 32]
            masks.append(_lib.gemm_upscale_mask(up1, p["up2_w"], p["up2_b"], hyper, h, w))
        masks = torch.stack(masks, dim=1) if len(masks) > 1 else masks[0].unsqueeze(1)
        iou = iou[:, 1:] if multimask_output else iou[:, 0:1]
        return masks, iou

    def forward(self, image_embeddings, image_positional_embeddings, sparse_prompt_embeddings,
                dense_prompt_embeddings, multimask_output, attention_similarity=None,
                target_embedding=None, output_attentions=None):
        """Reference signature (HF:461-470 + the 3-tuple of transformers 4.38 the callers unpack,
        M:369, M:1685).  Per-prompt NCHW inputs; point_batch_size must be 1."""
        if attention_similarity is not None or target_embedding is not None:
            raise NotImplementedError("attention_similarity / target_embedding are not used by RSPrompter")
        N, C, h, w = image_embeddings.shape
        assert sparse_prompt_embeddings.shape[1] == 1, "point_batch_size must be 1"
        to_rows = lambda t: t.to(torch.float32).permute(0, 2, 3, 1).reshape(-1, C).contiguous()  # noqa: E731
        pos_rows = to_rows(image_positional_embeddings[:1])
        masks, iou = self.decode(to_rows(image_embeddings), pos_rows, sparse_prompt_embeddings[:, 0],
                                 (h, w), dense_rows=to_rows(dense_prompt_embeddings),
                                 multimask_output=multimask_output)
        return masks.unsqueeze(1), iou.unsqueeze(1), None


@MODELS.register_module(force=True)
class RSSamMaskDecoder(BaseModule):
    """Drop-in for mmdet.rsprompter RSSamMaskDecoder (M:899-914)."""

    def __init__(self, hf_pretrain_name, extra_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        self.mask_decoder = SamMaskDecoderB200(decoder_arch(hf_pretrain_name, extra_config))
        _load_pretrained(self.mask_decoder, init_cfg, [(r"^module\.", ""), (r"^mask_decoder\.", "")])

    def init_weights(self):
        pass

    def forward(self, *args, **kwargs):
        return self.mask_decoder(*args, **kwargs)


class SamPositionalEmbeddingB200(nn.Module):
    """HF SamPositionalEmbedding (HF:546-566): random-Fourier features of normalised coordinates.

    The image-wide table (M:85-95) depends only on the grid size, so it is evaluated once per
    size and cached; it is constant folding at set-up, not per-batch work."""

    def __init__(self, num_pos_feats: int = 128, scale: float = 1.0):
        super().__init__()
        self.scale = scale
        self.positional_embedding = nn.Parameter(scale * torch.randn(2, num_pos_feats), requires_grad=False)
        self._cache: dict = {}

    def forward(self, input_coords, input_shape=None):
        c = input_coords.clone()
        if input_shape is not None:
            c[..., 0] = c[..., 0] / input_shape[1]
            c[..., 1] = c[..., 1] / input_shape[0]
        c = (2 * c - 1).to(self.positional_embedding.dtype) @ self.positional_embedding
        c = 2 * math.pi * c
        return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)

    def image_wide_rows(self, size: int) -> torch.Tensor:
        """fp32 [size*size, 2F] channels-last rows of get_image_wide_positional_embeddings (M:85-95)."""
        key = (size, self.positional_embedding.device, self.positional_embedding._version)
        if key not in self._cache:
            g = torch.ones(size, size, device=self.positional_embedding.device, dtype=torch.float32)
            y = (g.cumsum(0) - 0.5) / size
            x = (g.cumsum(1) - 0.5) / size
            self._cache = {key: self.forward(torch.stack([x, y], dim=-1)).reshape(size * size, -1).contiguous()}
        return self._cache[key]


@MODELS.register_module(force=True)
class RSSamPositionalEmbedding(BaseModule):
    """Drop-in for RSSamPositionalEmbedding (M:744-759)."""

    def __init__(self, hf_pretrain_name, extra_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        va = vision_arch(hf_pretrain_name, extra_config)
        self.shared_image_embedding = SamPositionalEmbeddingB200(va.num_pos_feats, va.pe_scale())
        _load_pretrained(self.shared_image_embedding, init_cfg,
                         [(r"^module\.", ""), (r"^shared_image_embedding\.", "")])

    def init_weights(self):
        pass

    def forward(self, *args, **kwargs):
        return self.shared_image_embedding(*args, **kwargs)


class _MaskEmbed(nn.Module):
    """Parameter tree of HF SamMaskEmbedding (HF:569-593)."""

    def __init__(self, a: SamDecoderArch):
        super().__init__()
        mc = a.mask_input_channels
        self.conv1 = _Affine((mc // 4, 1, 2, 2))
        self.conv2 = _Affine((mc, mc // 4, 2, 2))
        self.conv3 = _Affine((a.hidden_size, mc, 1, 1))
        self.layer_norm1 = _Affine((mc // 4,))
        self.layer_norm2 = _Affine((mc,))


class SamPromptEncoderB200(nn.Module):
    """The members of HF SamPromptEncoder the RSPrompter heads touch (M:305-307, M:1635)."""

    def __init__(self, a: SamDecoderArch):
        super().__init__()
        self.no_mask_embed = _Embedding(1, a.hidden_size)
        self.mask_embed = _MaskEmbed(a)


@MODELS.register_module(force=True)
class RSSamPromptEncoder(BaseModule):
    """Drop-in for RSSamPromptEncoder (M:881-896)."""

    def __init__(self, hf_pretrain_name, extra_config=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        self.prompt_encoder = SamPromptEncoderB200(decoder_arch(hf_pretrain_name, extra_config))
        _load_pretrained(self.prompt_encoder, init_cfg, [(r"^module\.", ""), (r"^prompt_encoder\.", "")])

    def init_weights(self):
        pass


__all__ = ["SamMaskDecoderB200", "RSSamMaskDecoder", "RSSamPositionalEmbedding", "RSSamPromptEncoder",
           "SamPositionalEmbeddingB200", "SamPromptEncoderB200"]
