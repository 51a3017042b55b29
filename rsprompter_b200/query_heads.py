"""RSPrompter-query heads on the H100 kernels: MSDeformAttnPixelDecoder -> Mask2Former transformer decoder
-> RSMask2FormerHead (SAM decoder prompted by the queries) -> RSMaskFormerFusionHead (M:274-715;
mmdet/models/layers/msdeformattn_pixel_decoder.py:21-246; layers/transformer/mask2former_layers.py:9-135;
seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py:126-182).

All Linear / conv layers are tensor-core GEMMs; the positional terms never cost an add pass:
``(x + pos) W^T = x W^T + pos W^T`` and ``pos W^T`` (a constant of the weights and the map size) enters as a
broadcast residual of the GEMM epilogue; LayerNorms after out_proj / FFN are the row-LN epilogue.
With ``decoder_plus=True`` (every shipped query config) the attention masks of the next layer come from
``mask_pred_plus`` and ``predict`` reads only the last layer's masks (M:380-385, 644-645), so the SAM mask
decoder runs once (after the last layer) instead of 7 times: output-identical, 6/7 of hot loop #3 removed.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib
from .anchor_heads import sine_pe_rows
from .necks import _PrepMixin, _conv, conv1x1, conv3x3, prep_conv
from .registry import MODELS, BaseModule, ConfigDict, InstanceData
from .sam_encoder import _Affine


def _cfg(d):
    """Nested dict -> ConfigDict (attribute access at every level)."""
    if isinstance(d, dict):
        return ConfigDict({k: _cfg(v) for k, v in d.items()})
    if d is None:
        return ConfigDict()
    return d


class _Emb(nn.Module):
    def __init__(self, n: int, c: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n, c), requires_grad=False)


class _ConvGN(nn.Module):
    """mmcv ConvModule(norm_cfg=GN): conv (+bias when asked) -> GroupNorm (-> ReLU)."""

    def __init__(self, cin: int, cout: int, k: int, bias: bool):
        super().__init__()
        self.conv = _conv(cout, cin, k, bias=bias)
        self.gn = _Affine((cout,))


class _MSDeformAttn(nn.Module):
    def __init__(self, E: int, heads: int, levels: int, points: int):
        super().__init__()
        self.sampling_offsets = _Affine((heads * levels * points * 2, E))
        self.attention_weights = _Affine((heads * levels * points, E))
        self.value_proj = _Affine((E, E))
        self.output_proj = _Affine((E, E))


class _FFN(nn.Module):
    def __init__(self, E: int, F: int):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(_Affine((F, E))), _Affine((E, F)))


class _EncLayer(nn.Module):
    def __init__(self, E, heads, levels, points, F):
        super().__init__()
        self.self_attn = _MSDeformAttn(E, heads, levels, points)
        self.ffn = _FFN(E, F)
        self.norms = nn.ModuleList([_Affine((E,)), _Affine((E,))])


class _Encoder(nn.Module):
    def __init__(self, n, E, heads, levels, points, F):
        super().__init__()
        self.layers = nn.ModuleList(_EncLayer(E, heads, levels, points, F) for _ in range(n))


class _TorchMHA(nn.Module):
    def __init__(self, E: int):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * E, E), requires_grad=False)
        self.in_proj_bias = nn.Parameter(torch.empty(3 * E), requires_grad=False)
        self.out_proj = _Affine((E, E))


class _MHA(nn.Module):
    def __init__(self, E: int):
        super().__init__()
        self.attn = _TorchMHA(E)


class _DecLayer(nn.Module):
    def __init__(self, E, F):
        super().__init__()
        self.self_attn = _MHA(E)
        self.cross_attn = _MHA(E)
        self.ffn = _FFN(E, F)
        self.norms = nn.ModuleList([_Affine((E,)) for _ in range(3)])


class _Decoder(nn.Module):
    def __init__(self, n, E, F):
        super().__init__()
        self.layers = nn.ModuleList(_DecLayer(E, F) for _ in range(n))
        self.post_norm = _Affine((E,))


def _bf(t):
    return t.detach().to(torch.bfloat16).contiguous()


def _f32(t):
    return t.detach().float().contiguous()


@MODELS.register_module(force=True)
class MSDeformAttnPixelDecoder(_PrepMixin, BaseModule):
    def __init__(self, in_channels=(256, 512, 1024, 2048), strides=(4, 8, 16, 32), feat_channels=256, out_channels=256,
                 num_outs=3, norm_cfg=None, act_cfg=None, encoder=None, positional_encoding=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        enc = _cfg(encoder)
        sa = enc.layer_cfg.self_attn_cfg
        assert norm_cfg is not None and norm_cfg.get("type") == "GN" and feat_channels in (128, 256) and sa.num_heads == 8
        self.num_input_levels, self.num_encoder_levels = len(in_channels), sa.num_levels
        self.num_points, self.num_outs, self.E = sa.num_points, num_outs, feat_channels
        self.groups = norm_cfg.get("num_groups", 32)
        E, L = feat_channels, self.num_encoder_levels
        self.input_convs = nn.ModuleList(_ConvGN(in_channels[self.num_input_levels - 1 - i], E, 1, True) for i in range(L))
        self.encoder = _Encoder(enc.num_layers, E, sa.num_heads, L, sa.num_points,
                                enc.layer_cfg.ffn_cfg.feedforward_channels)
        self.level_encoding = _Emb(L, E)
        n_fpn = self.num_input_levels - L
        self.lateral_convs = nn.ModuleList(_ConvGN(in_channels[i], E, 1, False) for i in range(n_fpn))
        self.output_convs = nn.ModuleList(_ConvGN(E, E, 3, False) for _ in range(n_fpn))
        self.mask_feature = _conv(out_channels, E, 1)
        self._init_prep()
        self._const: dict = {}

    @torch.no_grad()
    def _prepare(self):
        p = dict(inp=[], enc=[], lat=[], out=[])
        for m in self.input_convs:
            p["inp"].append((*prep_conv(m.conv.weight, m.conv.bias), _f32(m.gn.weight), _f32(m.gn.bias)))
        for l in self.encoder.layers:
            sa = l.self_attn
            wow = torch.cat([sa.sampling_offsets.weight, sa.attention_weights.weight], dim=0)
            bow = torch.cat([sa.sampling_offsets.bias, sa.attention_weights.bias], dim=0)
            p["enc"].append(dict(wow=_bf(wow), wow32=_f32(wow), bow=_f32(bow), wv=_bf(sa.value_proj.weight),
                                 bv=_f32(sa.value_proj.bias), wo=_bf(sa.output_proj.weight), bo=_f32(sa.output_proj.bias),
                                 n0=(_f32(l.norms[0].weight), _f32(l.norms[0].bias)),
                                 n1=(_f32(l.norms[1].weight), _f32(l.norms[1].bias)),
                                 w1=_bf(l.ffn.layers[0][0].weight), b1=_f32(l.ffn.layers[0][0].bias),
                                 w2=_bf(l.ffn.layers[1].weight), b2=_f32(l.ffn.layers[1].bias)))
        for m in self.lateral_convs:
            p["lat"].append((prep_conv(m.conv.weight, None)[0], _f32(m.gn.weight), _f32(m.gn.bias)))
        for m in self.output_convs:
            p["out"].append((prep_conv(m.conv.weight, None)[0], _f32(m.gn.weight), _f32(m.gn.bias)))
        p["mf"] = prep_conv(self.mask_feature.weight, self.mask_feature.bias)
        self._prep = p
        self._const = {}
        return p

    def _pos_terms(self, shapes: list, device):
        """Per size: concatenated (sine PE + level encoding) rows and, per encoder layer, their projection
        through [sampling_offsets | attention_weights] plus the bias (broadcast residual of that GEMM)."""
        key = (tuple(shapes), str(device))
        if key not in self._const:
            p = self._prep
            rows = []
            for i, (h, w) in enumerate(shapes):
                pe = sine_pe_rows(h, w, self.E // 2, device)[0].permute(1, 2, 0).reshape(h * w, self.E)
                rows.append(pe + self.level_encoding.weight[i].float().view(1, -1))
            pos = torch.cat(rows, dim=0).contiguous()
            pw = [(pos @ e["wow32"].t() + e["bow"]).contiguous() for e in p["enc"]]
            self._const[key] = (pos, pw)
        return self._const[key]

    @torch.no_grad()
    def forward_nhwc(self, feats: list):
        """feats: 5 bf16 NHWC levels (high -> low resolution).
        -> (mask_feature bf16 [B, H0, W0, out], [memories bf16 [B, h, w, E]] low -> high resolution)."""
        p = self._prep or self._prepare()
        nl, L, E = self.num_input_levels, self.num_encoder_levels, self.E
        B = feats[0].shape[0]
        xs, shapes = [], []
        for i in range(L):
            f = feats[nl - 1 - i]
            w, b, g, be = p["inp"][i]
            y = _lib.groupnorm_nhwc(conv1x1(f, w, b), g, be, self.groups)
            xs.append(y.view(B, -1, E))
            shapes.append((f.shape[1], f.shape[2]))
        x = torch.cat(xs, dim=1).contiguous()                       # [B, NQ, E] bf16
        NQ = x.shape[1]
        _, pws = self._pos_terms(shapes, x.device)
        x = x.view(B * NQ, E)
        for e, pw in zip(p["enc"], pws):
            ow = _lib.gemm(x, e["wow"], None, residual=pw, res_mod=NQ, out_dtype=torch.float32)
            val = _lib.gemm(x, e["wv"], e["bv"])
            samp = _lib.ms_deform_attn_sample(val.view(B, NQ, E), ow, shapes, self.num_points)
            x = _lib.gemm(samp, e["wo"], e["bo"], residual=x, ln=(*e["n0"], 1e-5))
            hdn = _lib.gemm(x, e["w1"], e["b1"], act="relu")
            x = _lib.gemm(hdn, e["w2"], e["b2"], residual=x, ln=(*e["n1"], 1e-5))
        mem = x.view(B, NQ, E)
        outs, start = [], 0
        for (h, w) in shapes:
            outs.append(mem[:, start:start + h * w].contiguous().view(B, h, w, E))
            start += h * w
        for i in range(nl - L - 1, -1, -1):
            wl, gl, bl = p["lat"][i]
            y = _lib.groupnorm_nhwc(conv1x1(feats[i], wl, None), gl, bl, self.groups, up=outs[-1])
            wo, go, bo = p["out"][i]
            outs.append(_lib.groupnorm_nhwc(conv3x3(y, wo, None), go, bo, self.groups, relu=True))
        mask_feature = conv1x1(outs[-1], *p["mf"])
        return mask_feature, outs[:self.num_outs]


@MODELS.register_module(force=True)
class RSMask2FormerHead(_PrepMixin, BaseModule):
    """M:274-658 (inference half) over Mask2FormerHead (dense_heads/mask2former_head.py:24-156)."""

    def __init__(self, mask_decoder, decoder_plus, with_sincos=True, per_pointset_point=1, multimask_output=False,
                 attention_similarity=None, target_embedding=None, output_attentions=None, in_channels=None,
                 feat_channels=128, out_channels=256, num_things_classes=80, num_stuff_classes=0, num_queries=100,
                 num_transformer_feat_level=3, pixel_decoder=None, enforce_decoder_input_project=False,
                 transformer_decoder=None, positional_encoding=None, loss_cls=None, loss_mask=None, loss_dice=None,
                 train_cfg=None, test_cfg=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        assert decoder_plus, "decoder_plus=False is not shipped by any RSPrompter config"
        assert not enforce_decoder_input_project and feat_channels == 128 and out_channels == 256
        td = _cfg(transformer_decoder)
        self.num_classes = num_things_classes + num_stuff_classes
        self.num_queries, self.num_levels = num_queries, num_transformer_feat_level
        self.feat_channels, self.out_channels = feat_channels, out_channels
        self.per_pointset_point, self.with_sincos, self.multimask_output = per_pointset_point, with_sincos, multimask_output
        self.num_layers = td.num_layers
        E = feat_channels
        pd = dict(pixel_decoder)
        pd.update(in_channels=in_channels, feat_channels=feat_channels, out_channels=out_channels)
        self.pixel_decoder = MODELS.build(pd)
        self.transformer_decoder = _Decoder(td.num_layers, E, td.layer_cfg.ffn_cfg.feedforward_channels)
        self.query_embed, self.query_feat = _Emb(num_queries, E), _Emb(num_queries, E)
        self.level_embed = _Emb(num_transformer_feat_level, E)
        self.cls_embed = nn.Sequential(_Affine((E, E)), nn.Identity(), _Affine((self.num_classes + 1, E)))
        self.mask_embed = nn.Sequential(_Affine((E, E)), nn.Identity(), _Affine((E, E)), nn.Identity(),
                                        _Affine((out_channels, E)))
        ns = 2 if with_sincos else 1
        self.point_emb = nn.Sequential(_Affine((E // 2, E)), nn.Identity(), _Affine((E // 2, E // 2)), nn.Identity(),
                                       _Affine((out_channels * ns * per_pointset_point, E // 2)))
        self.mask_decoder = MODELS.build(mask_decoder)
        pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name=mask_decoder.get("hf_pretrain_name"),
                               init_cfg=mask_decoder.get("init_cfg")))
        self.sam_mask_embed = pe.prompt_encoder.mask_embed
        self._init_prep()
        self._const: dict = {}

    def init_weights(self):
        pass

    @torch.no_grad()
    def _prepare(self):
        E = self.feat_channels
        lin = lambda m: (_bf(m.weight), _f32(m.bias))  # noqa: E731
        layers = []
        for l in self.transformer_decoder.layers:
            d = {}
            for name, mod in (("ca", l.cross_attn.attn), ("sa", l.self_attn.attn)):
                W, b = mod.in_proj_weight, mod.in_proj_bias
                d[name] = dict(wq=_bf(W[:E]), bq=_f32(b[:E]), wk=_bf(W[E:2 * E]), bk=_f32(b[E:2 * E]), wv=_bf(W[2 * E:]),
                               bv=_f32(b[2 * E:]), wqk=_bf(W[:2 * E]), bqk=_f32(b[:2 * E]), w32=_f32(W),
                               wo=_bf(mod.out_proj.weight), bo=_f32(mod.out_proj.bias))
            d["norms"] = [(_f32(n.weight), _f32(n.bias)) for n in l.norms]
            d["w1"], d["b1"] = lin(l.ffn.layers[0][0])
            d["w2"], d["b2"] = lin(l.ffn.layers[1])
            layers.append(d)
        me = self.sam_mask_embed
        self._prep = dict(
            layers=layers, post=(_f32(self.transformer_decoder.post_norm.weight), _f32(self.transformer_decoder.post_norm.bias)),
            cls=[lin(self.cls_embed[0]), lin(self.cls_embed[2])],
            mask=[lin(self.mask_embed[i]) for i in (0, 2, 4)], pts=[lin(self.point_emb[i]) for i in (0, 2, 4)],
            sam_me=[_f32(t) for t in (me.conv1.weight, me.conv1.bias, me.layer_norm1.weight, me.layer_norm1.bias,
                                      me.conv2.weight, me.conv2.bias, me.layer_norm2.weight, me.layer_norm2.bias,
                                      me.conv3.weight.reshape(self.out_channels, -1), me.conv3.bias)],
            qe=_f32(self.query_embed.weight), qf=_f32(self.query_feat.weight), le=_f32(self.level_embed.weight))
        self._const = {}
        return self._prep

    def _level_consts(self, shapes: list, device):
        """Weight- and size-dependent constants: per decoder layer the key-side positional projection
        (pos + level_embed) Wk^T, the value bias bv + level_embed Wv^T and the query_embed projections."""
        key = (tuple(shapes), str(device))
        if key not in self._const:
            p, E = self._prep, self.feat_channels
            pos = [sine_pe_rows(h, w, E // 2, device)[0].permute(1, 2, 0).reshape(h * w, E) for h, w in shapes]
            out = []
            for i, d in enumerate(p["layers"]):
                lvl = i % self.num_levels
                ca, sa = d["ca"], d["sa"]
                W = ca["w32"]
                le = p["le"][lvl].view(1, -1)
                out.append(dict(pk=((pos[lvl] + le) @ W[E:2 * E].t()).contiguous(),
                                bv=(ca["bv"] + (le @ W[2 * E:].t()).view(-1)).contiguous(),
                                qe_q=(p["qe"] @ W[:E].t()).contiguous(),
                                qe_qk=(p["qe"] @ sa["w32"][:2 * E].t()).contiguous()))
            self._const[key] = out
        return self._const[key]

    def _mlp(self, x_bf: torch.Tensor, layers: list, out_dtype=torch.bfloat16, out=None, row_map=None) -> torch.Tensor:
        h = x_bf
        for w, b in layers[:-1]:
            h = _lib.gemm(h, w, b, act="relu")
        if out is not None:
            return _lib.gemm(h, *layers[-1], out=out, row_map=row_map)
        return _lib.gemm(h, *layers[-1], out_dtype=out_dtype)

    def _padded_queries(self, B: int, nq: int, C: int, device):
        """Per-image 128-row blocks for the grouped  mask_embed x mask_feature  products (one launch for all images):
        -> (zero-initialised bf16 [B*128, C] buffer, scatter map compact row -> padded row, map padded -> compact / -1)."""
        key = ("mepad", B, nq, C, str(device))
        if key not in self._const:
            q = torch.arange(nq, device=device, dtype=torch.int32)
            b = torch.arange(B, device=device, dtype=torch.int32)
            scat = (b.view(B, 1) * 128 + q.view(1, nq)).reshape(-1).contiguous()
            back = torch.full((B, 128), -1, device=device, dtype=torch.int32)
            back[:, :nq] = b.view(B, 1) * nq + q.view(1, nq)
            self._const[key] = (torch.zeros(B * 128, C, device=device, dtype=torch.bfloat16), scat, back.reshape(-1).contiguous())
        return self._const[key]

    @torch.no_grad()
    def forward_nhwc(self, feats: list, emb_rows: torch.Tensor, pos_rows: torch.Tensor, emb_hw: tuple,
                     capture: dict | None = None):
        """-> cls fp32 [B, nq, C+1], mask_pred fp32 [B*nq, 256, 256] (SAM decoder), mask_pred_plus fp32 [B, nq, H0, W0]."""
        p = self._prep or self._prepare()
        E, nq, B = self.feat_channels, self.num_queries, feats[0].shape[0]
        mask_feature, mems = self.pixel_decoder.forward_nhwc(feats)
        H0, W0 = mask_feature.shape[1], mask_feature.shape[2]
        shapes = [(m.shape[1], m.shape[2]) for m in mems[:self.num_levels]]
        consts = self._level_consts(shapes, mask_feature.device)
        mem_rows = [m.reshape(B * m.shape[1] * m.shape[2], E) for m in mems[:self.num_levels]]
        mf_rows = mask_feature.view(B, H0 * W0, -1)
        qf = p["qf"].unsqueeze(0).expand(B, -1, -1).reshape(B * nq, E).contiguous()      # fp32 query stream

        # F.interpolate(mask_pred_plus, level size) = mask_embed x resize(mask_feature)^T (bilinear is linear):
        # the intermediate layers only ever need level-sized logits, never the H0 x W0 maps (M:386-392)
        mf_lvl = [_lib.resize_bilinear_nhwc(mask_feature, s).view(B, s[0] * s[1], -1) for s in shapes]

        grouped = nq <= 128
        if grouped:
            me_pad, scat, back = self._padded_queries(B, nq, self.out_channels, mask_feature.device)

        def head(qf32: torch.Tensor, lvl: int, final: bool):
            x = _lib.layernorm(qf32, *p["post"], 1e-5)                                    # post_norm -> bf16
            if grouped:      # mask_embed rows of image b land in rows [128 b, 128 b + nq) of a zero-padded buffer
                self._mlp(x, p["mask"], out=me_pad, row_map=scat)
                me_of = lambda b: me_pad[b * 128:b * 128 + nq]  # noqa: E731
            else:
                me = self._mlp(x, p["mask"])                                              # [B*nq, 256]
                me_of = lambda b: me[b * nq:(b + 1) * nq]  # noqa: E731
            if not final:
                hw_l = mf_lvl[lvl].shape[1]
                logits = torch.empty(B * nq, hw_l, device=x.device, dtype=torch.float32)
                if grouped:  # one grouped GEMM for all images: row block b multiplies its own image's features
                    _lib.gemm_grouped(me_pad, mf_lvl[lvl].reshape(B * hw_l, -1), logits, hw_l, 128, hw_l, row_map=back)
                else:
                    for b in range(B):
                        _lib.gemm(me_of(b), mf_lvl[lvl][b], None, out=logits[b * nq:(b + 1) * nq])
                return _lib.attn_mask_bits(logits), None, None, None
            mpp = torch.empty(B, nq, H0 * W0, device=x.device, dtype=torch.float32)
            for b in range(B):                                                            # einsum 'bqc,bchw->bqhw'
                _lib.gemm(me_of(b), mf_rows[b], None, out=mpp[b])
            cls = self._mlp(x, p["cls"], out_dtype=torch.float32)
            pts = self._mlp(x, p["pts"], out_dtype=torch.float32).view(B * nq, self.per_pointset_point, -1)
            sparse = _lib.sin_fold(pts.contiguous()) if self.with_sincos else pts
            return None, mpp.view(B * nq, H0, W0), cls, sparse

        attn_mask, mpp, cls, sparse = head(qf, 0, final=self.num_layers == 0)
        for i, d in enumerate(p["layers"]):
            lvl = i % self.num_levels
            hw = shapes[lvl][0] * shapes[lvl][1]
            c = consts[i]
            ca, sa = d["ca"], d["sa"]
            qb = _lib.cast_bf16(qf)
            Q = _lib.gemm(qb, ca["wq"], ca["bq"], residual=c["qe_q"], res_mod=nq)
            K = _lib.gemm(mem_rows[lvl], ca["wk"], ca["bk"], residual=c["pk"], res_mod=hw)
            V = _lib.gemm(mem_rows[lvl], ca["wv"], c["bv"])
            att = _lib.mha_small(Q, K, V, B, nq, hw, mask=attn_mask)
            qf = _lib.gemm(att, ca["wo"], ca["bo"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][0], 1e-5))
            qb = _lib.cast_bf16(qf)
            QK = _lib.gemm(qb, sa["wqk"], sa["bqk"], residual=c["qe_qk"], res_mod=nq)      # [B*nq, 2E]
            Vs = _lib.gemm(qb, sa["wv"], sa["bv"])
            att = _lib.mha_small(QK[:, :E], QK[:, E:], Vs, B, nq, nq)
            qf = _lib.gemm(att, sa["wo"], sa["bo"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][1], 1e-5))
            hdn = _lib.gemm(_lib.cast_bf16(qf), d["w1"], d["b1"], act="relu")
            qf = _lib.gemm(hdn, d["w2"], d["b2"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][2], 1e-5))
            last = i == self.num_layers - 1
            attn_mask, mpp, cls, sparse = head(qf, (i + 1) % self.num_levels, final=last)
        # the single live SAM-decoder invocation (M:359-378 of the last _forward_head)
        h, w = emb_hw
        src_pair = _lib.mask_embed_src(mpp, p["sam_me"], emb_rows, pos_rows, nq, (h, w))
        masks, _ = self.mask_decoder.mask_decoder.decode(None, pos_rows, sparse, (h, w), src_pair=src_pair,
                                                         multimask_output=self.multimask_output)
        if capture is not None:
            capture.update(mask_feature=mask_feature, memories=mems, sparse=sparse)
        return cls.view(B, nq, -1), masks[:, 0].contiguous(), mpp.view(B, nq, H0, W0)


@MODELS.register_module(force=True)
class RSMaskFormerFusionHead(BaseModule):
    """M:661-715 + MaskFormerFusionHead.instance_postprocess / panoptic_postprocess (maskformer_fusion_head.py:126-182,
    41-106)."""

    def __init__(self, num_things_classes=80, num_stuff_classes=0, test_cfg=None, loss_panoptic=None, init_cfg=None,
                 **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        self.num_things_classes, self.num_stuff_classes = num_things_classes, num_stuff_classes
        self.num_classes = num_things_classes + num_stuff_classes
        self.test_cfg = _cfg(test_cfg)

    @torch.no_grad()
    def instance_postprocess_batched(self, cls: torch.Tensor, mask_pred: torch.Tensor, size: tuple, metas: list | None = None,
                                     rescale: bool = True):
        """cls fp32 [B, nq, C+1]; mask_pred fp32 [B*nq, hm, wm] low-res logits (the bilinear up-sampling of
        M:652-656 and the crop / rescale of M:679-691 are fused into the mask kernel).
        -> dict of per-image lists / [B, K, ...] tensors (all images at the batch shape: stacked tensors)."""
        B, nq, _ = cls.shape
        C = self.num_classes
        K = int(self.test_cfg.get("max_per_image", 100))
        scores = torch.softmax(cls, dim=-1)[:, :, :-1].reshape(B, nq * C)
        sc, top = scores.topk(K, dim=1, sorted=False)
        labels = top % C
        query = top // C
        sel = (query + torch.arange(B, device=cls.device).view(B, 1) * nq).to(torch.int32).contiguous()
        keep_thing = labels < self.num_things_classes
        if metas is None or all(m is None for m in metas):
            masks, det, boxes = _lib.query_postprocess(mask_pred, sel.reshape(-1), sc.reshape(-1).contiguous(), size)
            return dict(masks=masks.view(B, K, *size), scores=det.view(B, K), bboxes=boxes.view(B, K, 4), labels=labels,
                        query=query, is_thing=keep_thing)
        ms, ds, bs = [], [], []
        for b, m in enumerate(metas):      # image sizes differ: one launch pair per image, no host sync
            geom = dict(size=size) if m is None else \
                dict(rescale=(size, m["crop_hw"], m["ori_hw"] if rescale else m["crop_hw"]))
            mk, det, bx = _lib.query_postprocess(mask_pred, sel[b].contiguous(), sc[b].contiguous(), **geom)
            ms.append(mk); ds.append(det); bs.append(bx)
        return dict(masks=ms, scores=ds, bboxes=bs, labels=labels, query=query, is_thing=keep_thing)

    @torch.no_grad()
    def panoptic_postprocess_batched(self, cls: torch.Tensor, mask_pred: torch.Tensor, size: tuple,
                                     metas: list | None = None, rescale: bool = True):
        """MaskFormerFusionHead.panoptic_postprocess (maskformer_fusion_head.py:41-106) of every image, on the masks
        instance_postprocess_batched resamples (M:652-656 up-sampling, M:679-691 crop / rescale), with no host read.
        cls fp32 [B, nq, C+1]; mask_pred fp32 [B*nq, hm, wm] low-res logits -> (per-image int32 [1, H, W] maps,
        per-image dicts of the per-query mask_area / original_area / segment_id, int32 [nq])."""
        B, nq, _ = cls.shape
        _lib.check_panoptic_bounds(nq, self.num_classes)
        cfg = self.test_cfg
        thr = float(cfg.get("object_mask_thr", 0.8))
        args = (self.num_things_classes, self.num_classes, float(cfg.get("iou_thr", 0.8)),
                bool(cfg.get("filter_low_score", False)))
        scores, labels = torch.softmax(cls, dim=-1).max(-1)
        keep = labels.ne(self.num_classes) & (scores > thr)
        if metas is None or all(m is None for m in metas):
            pan, st = _lib.panoptic_postprocess(mask_pred, keep, scores, labels, *args, size=size)
            return list(pan), [{k: v[b] for k, v in st.items()} for b in range(B)]
        pans, stats = [], []
        for b, m in enumerate(metas):      # image sizes differ: one launch triple per image, no host sync
            geom = dict(size=size) if m is None else \
                dict(rescale=(size, m["crop_hw"], m["ori_hw"] if rescale else m["crop_hw"]))
            pan, st = _lib.panoptic_postprocess(mask_pred[b * nq:(b + 1) * nq], keep[b:b + 1], scores[b:b + 1],
                                                labels[b:b + 1], *args, **geom)
            pans.append(pan[0])
            stats.append({k: v[0] for k, v in st.items()})
        return pans, stats

    @torch.no_grad()
    def instance_postprocess_record(self, cls: torch.Tensor, mask_pred: torch.Tensor, rec, metas: list | None = None,
                                    size: tuple | None = None) -> None:
        """instance_postprocess for images at the batch shape (4x the logit size), written into a ResultRecord: the
        masks go out bit-packed, rows = (tight box, cls * mask score, label) (maskformer_fusion_head.py:149-182).
        With ``metas`` (per-image dict(ori_hw, crop_hw) of resized images, batch shape ``size``) the masks, scores and
        boxes are those of instance_postprocess_batched(rescale=True), written at ori_hw."""
        B, nq, _ = cls.shape
        C = self.num_classes
        K = rec.slots
        assert self.num_stuff_classes == 0, "records hold fixed-size instance lists (no stuff filtering)"
        scores = torch.softmax(cls, dim=-1)[:, :, :-1].reshape(B, nq * C)
        sc, top = scores.topk(K, dim=1, sorted=False)
        labels, query = top % C, top // C
        sel = (query + torch.arange(B, device=cls.device).view(B, 1) * nq).to(torch.int32).contiguous()
        if metas is not None:
            bits = rec.mask_bits.view(B * K, *rec.mask_bits.shape[2:])
            det = torch.empty(B, K, device=cls.device, dtype=torch.float32)
            boxes = torch.empty(B, K, 4, device=cls.device, dtype=torch.float32)
            for b, m in enumerate(metas):
                _lib.query_postprocess(mask_pred, sel[b].contiguous(), sc[b].contiguous(),
                                       rescale=(size, m["crop_hw"], m["ori_hw"]), bits=bits[b * K:(b + 1) * K],
                                       scores=det[b], boxes=boxes[b])
            torch.cat([boxes, det[..., None], labels.to(torch.float32)[..., None]], dim=2, out=rec.rows)
            rec.counts.fill_(K)
            return
        _, det, boxes = _lib.query_postprocess(mask_pred, sel.reshape(-1), sc.reshape(-1).contiguous(),
                                               bits=rec.mask_bits.view(B * K, rec.hw[0], rec.hw[1] // 8))
        torch.cat([boxes.view(B, K, 4), det.view(B, K, 1), labels.to(torch.float32)[..., None]], dim=2, out=rec.rows)
        rec.counts.fill_(K)


@MODELS.register_module(force=True)
class Mask2FormerHead(_PrepMixin, BaseModule):
    """The stock mmdet Mask2FormerHead (dense_heads/mask2former_head.py:24-156 build, :340-380 _forward_head, :382-460
    forward; inference half) as SAMSegMask2Former uses it (configs/rsprompter/_base_/samseg-mask2former.py:86-160):
    feat_channels 256 (8 heads x 32), 9 decoder layers, cls_embed = one Linear, masks = mask_embed x mask_feature.
    Same kernels and the same constant-folding of the positional terms as RSMask2FormerHead; the attention masks of the
    intermediate layers are formed at the level size from bilinearly resized mask features (F.interpolate is linear),
    so only the last layer materialises the H/4 x W/4 mask logits."""

    def __init__(self, in_channels=None, feat_channels=256, out_channels=256, num_things_classes=80,
                 num_stuff_classes=0, num_queries=100, num_transformer_feat_level=3, pixel_decoder=None,
                 enforce_decoder_input_project=False, transformer_decoder=None, positional_encoding=None, loss_cls=None,
                 loss_mask=None, loss_dice=None, train_cfg=None, test_cfg=None, init_cfg=None, **kwargs):
        BaseModule.__init__(self, init_cfg=None)
        td = _cfg(transformer_decoder)
        assert not enforce_decoder_input_project and feat_channels in (128, 256)
        assert td.layer_cfg.cross_attn_cfg.num_heads == 8 and td.layer_cfg.cross_attn_cfg.embed_dims == feat_channels
        self.num_classes = num_things_classes + num_stuff_classes
        self.num_queries, self.num_levels = num_queries, num_transformer_feat_level
        self.feat_channels, self.out_channels = feat_channels, out_channels
        self.num_layers = td.num_layers
        E = feat_channels
        pd = dict(pixel_decoder)
        pd.update(in_channels=in_channels, feat_channels=feat_channels, out_channels=out_channels)
        self.pixel_decoder = MODELS.build(pd)
        self.transformer_decoder = _Decoder(td.num_layers, E, td.layer_cfg.ffn_cfg.feedforward_channels)
        self.query_embed, self.query_feat = _Emb(num_queries, E), _Emb(num_queries, E)
        self.level_embed = _Emb(num_transformer_feat_level, E)
        self.cls_embed = _Affine((self.num_classes + 1, E))
        self.mask_embed = nn.Sequential(_Affine((E, E)), nn.Identity(), _Affine((E, E)), nn.Identity(),
                                        _Affine((out_channels, E)))
        self._init_prep()
        self._const: dict = {}

    def init_weights(self):
        pass

    _level_consts = RSMask2FormerHead._level_consts
    _mlp = RSMask2FormerHead._mlp
    _padded_queries = RSMask2FormerHead._padded_queries

    @torch.no_grad()
    def _prepare(self):
        E = self.feat_channels
        lin = lambda m: (_bf(m.weight), _f32(m.bias))  # noqa: E731
        layers = []
        for l in self.transformer_decoder.layers:
            d = {}
            for name, mod in (("ca", l.cross_attn.attn), ("sa", l.self_attn.attn)):
                W, b = mod.in_proj_weight, mod.in_proj_bias
                d[name] = dict(wq=_bf(W[:E]), bq=_f32(b[:E]), wk=_bf(W[E:2 * E]), bk=_f32(b[E:2 * E]), wv=_bf(W[2 * E:]),
                               bv=_f32(b[2 * E:]), wqk=_bf(W[:2 * E]), bqk=_f32(b[:2 * E]), w32=_f32(W),
                               wo=_bf(mod.out_proj.weight), bo=_f32(mod.out_proj.bias))
            d["norms"] = [(_f32(n.weight), _f32(n.bias)) for n in l.norms]
            d["w1"], d["b1"] = lin(l.ffn.layers[0][0])
            d["w2"], d["b2"] = lin(l.ffn.layers[1])
            layers.append(d)
        self._prep = dict(
            layers=layers, post=(_f32(self.transformer_decoder.post_norm.weight), _f32(self.transformer_decoder.post_norm.bias)),
            cls=[lin(self.cls_embed)], mask=[lin(self.mask_embed[i]) for i in (0, 2, 4)],
            qe=_f32(self.query_embed.weight), qf=_f32(self.query_feat.weight), le=_f32(self.level_embed.weight))
        self._const = {}
        return self._prep

    @torch.no_grad()
    def forward_nhwc(self, feats: list, capture: dict | None = None):
        """feats: the 5 bf16 NHWC neck levels -> cls fp32 [B, nq, C+1], mask logits fp32 [B*nq, H/4, W/4] (last layer)."""
        p = self._prep or self._prepare()
        E, nq, B = self.feat_channels, self.num_queries, feats[0].shape[0]
        hd = E // 8
        mask_feature, mems = self.pixel_decoder.forward_nhwc(feats)
        H0, W0 = mask_feature.shape[1], mask_feature.shape[2]
        shapes = [(m.shape[1], m.shape[2]) for m in mems[:self.num_levels]]
        consts = self._level_consts(shapes, mask_feature.device)
        mem_rows = [m.reshape(B * m.shape[1] * m.shape[2], E) for m in mems[:self.num_levels]]
        mf_rows = mask_feature.view(B, H0 * W0, -1)
        qf = p["qf"].unsqueeze(0).expand(B, -1, -1).reshape(B * nq, E).contiguous()      # fp32 query stream
        mf_lvl = [_lib.resize_bilinear_nhwc(mask_feature, s).view(B, s[0] * s[1], -1) for s in shapes]
        grouped = nq <= 128
        if grouped:
            me_pad, scat, back = self._padded_queries(B, nq, self.out_channels, mask_feature.device)

        def head(qf32: torch.Tensor, lvl: int, final: bool):
            x = _lib.layernorm(qf32, *p["post"], 1e-5)                                    # post_norm -> bf16
            if grouped:
                self._mlp(x, p["mask"], out=me_pad, row_map=scat)
                me_of = lambda b: me_pad[b * 128:b * 128 + nq]  # noqa: E731
            else:
                me = self._mlp(x, p["mask"])
                me_of = lambda b: me[b * nq:(b + 1) * nq]  # noqa: E731
            if not final:
                hw_l = mf_lvl[lvl].shape[1]
                logits = torch.empty(B * nq, hw_l, device=x.device, dtype=torch.float32)
                if grouped:
                    _lib.gemm_grouped(me_pad, mf_lvl[lvl].reshape(B * hw_l, -1), logits, hw_l, 128, hw_l, row_map=back)
                else:
                    for b in range(B):
                        _lib.gemm(me_of(b), mf_lvl[lvl][b], None, out=logits[b * nq:(b + 1) * nq])
                return _lib.attn_mask_bits(logits), None, None
            mp = torch.empty(B, nq, H0 * W0, device=x.device, dtype=torch.float32)
            for b in range(B):                                                            # einsum 'bqc,bchw->bqhw'
                _lib.gemm(me_of(b), mf_rows[b], None, out=mp[b])
            cls = self._mlp(x, p["cls"], out_dtype=torch.float32)
            return None, mp.view(B * nq, H0, W0), cls

        attn_mask, mp, cls = head(qf, 0, final=self.num_layers == 0)
        for i, d in enumerate(p["layers"]):
            lvl = i % self.num_levels
            hw = shapes[lvl][0] * shapes[lvl][1]
            c = consts[i]
            ca, sa = d["ca"], d["sa"]
            qb = _lib.cast_bf16(qf)
            Q = _lib.gemm(qb, ca["wq"], ca["bq"], residual=c["qe_q"], res_mod=nq)
            K = _lib.gemm(mem_rows[lvl], ca["wk"], ca["bk"], residual=c["pk"], res_mod=hw)
            V = _lib.gemm(mem_rows[lvl], ca["wv"], c["bv"])
            att = _lib.mha_small(Q, K, V, B, nq, hw, mask=attn_mask, head_dim=hd)
            qf = _lib.gemm(att, ca["wo"], ca["bo"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][0], 1e-5))
            qb = _lib.cast_bf16(qf)
            QK = _lib.gemm(qb, sa["wqk"], sa["bqk"], residual=c["qe_qk"], res_mod=nq)      # [B*nq, 2E]
            Vs = _lib.gemm(qb, sa["wv"], sa["bv"])
            att = _lib.mha_small(QK[:, :E], QK[:, E:], Vs, B, nq, nq, head_dim=hd)
            qf = _lib.gemm(att, sa["wo"], sa["bo"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][1], 1e-5))
            hdn = _lib.gemm(_lib.cast_bf16(qf), d["w1"], d["b1"], act="relu")
            qf = _lib.gemm(hdn, d["w2"], d["b2"], residual=qf, out_dtype=torch.float32, ln=(*d["norms"][2], 1e-5))
            attn_mask, mp, cls = head(qf, (i + 1) % self.num_levels, final=i == self.num_layers - 1)
        if capture is not None:
            capture.update(mask_feature=mask_feature, memories=mems)
        return cls.view(B, nq, -1), mp


@MODELS.register_module(force=True)
class MaskFormerFusionHead(RSMaskFormerFusionHead):
    """seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py (this repository's copy crops with the scaled original
    size exactly as M:679-691 does, :239-252): instance and panoptic post-processing shared with
    RSMaskFormerFusionHead."""


__all__ = ["MSDeformAttnPixelDecoder", "RSMask2FormerHead", "RSMaskFormerFusionHead", "Mask2FormerHead",
           "MaskFormerFusionHead"]
