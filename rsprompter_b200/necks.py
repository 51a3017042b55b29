"""RSFPN neck on the H100 kernels: RSFeatureAggregator / PseudoFeatureAggregator -> RSSimpleFPN
(M:917-1057, M:1277-1363), plus LN2d (M:32-50).

All feature maps are channels-last bf16 inside the pipeline (``forward_nhwc``); every conv is a
tensor-core GEMM: 1x1 directly on the pixel rows, 3x3 through ``rsp_im2col_nhwc``, the 2x2 / stride-2
transposed convs as four per-tap GEMMs whose epilogue scatters rows to the up-sampled grid
(``row_map``).  Eval-mode BatchNorm is folded into the conv weights when they are prepared; LN2d
over channels is the row LayerNorm kernel; the residual adds of the aggregator chain
(M:1051-1055) ride in the GEMM epilogues (ReLU is applied before the residual, as in the
reference).  ``forward`` keeps the reference's NCHW-in / NCHW-out signature.
"""
from __future__ import annotations

import torch
from torch import nn

from . import _lib
from .registry import MODELS, BaseModule
from .sam_encoder import _Affine


# ------------------------------------------------------------------------------ holders
class _BN(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c), requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(c), requires_grad=False)
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))
        self.eps = 1e-5


class _Slot(nn.Module):
    """Parameter-free placeholder (ReLU / GELU / Flatten positions in an nn.Sequential)."""


def _conv(cout: int, cin: int, k: int, bias: bool = True) -> _Affine:
    return _Affine((cout, cin, k, k), bias=bias)


class _ConvT(nn.Module):
    def __init__(self, cin: int, cout: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cin, cout, 2, 2), requires_grad=False)
        self.bias = nn.Parameter(torch.empty(cout), requires_grad=False)


@MODELS.register_module(force=True)
class LN2d(nn.Module):
    """Channel LayerNorm for NCHW tensors (M:32-50).  Inside the pipeline the data is channels-last
    and this is ``rsp_layernorm`` over rows; the module form keeps the reference's parameters."""

    def __init__(self, normalized_shape, eps=1e-6, requires_grad=True):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape), requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(normalized_shape), requires_grad=False)
        self.eps = eps
        self.normalized_shape = (normalized_shape,)

    def forward(self, x):
        B, C, H, W = x.shape
        rows = x.permute(0, 2, 3, 1).reshape(-1, C).contiguous().float()
        y = _lib.layernorm(rows, self.weight.float().contiguous(), self.bias.float().contiguous(), self.eps,
                           out_dtype=torch.float32)
        return y.view(B, H, W, C).permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------ weight prep
def fold_bn(w: torch.Tensor, b: torch.Tensor | None, bn: _BN | None):
    """conv -> eval BatchNorm folded into (w, b)."""
    w = w.detach().float()
    b = torch.zeros(w.shape[0], device=w.device) if b is None else b.detach().float()
    if bn is not None:
        s = bn.weight.detach().float() / torch.sqrt(bn.running_var.float() + bn.eps)
        w = w * s.view(-1, *([1] * (w.dim() - 1)))
        b = (b - bn.running_mean.float()) * s + bn.bias.detach().float()
    return w, b


def prep_conv(w: torch.Tensor, b: torch.Tensor | None, bn: _BN | None = None, pad_out: int = 0, pad_in: int = 0):
    """[Cout, Cin, kh, kw] -> bf16 [Cout(+pad), kh*kw*Cin(+pad)] (tap-major to match im2col) + fp32 bias.
    pad_in / pad_out: zero input / output channels up to that count (the padded output channels stay exactly 0 through
    bias-free ReLU stacks, which lets 32-channel maps ride in 64-channel buffers = one TMA swizzle atom)."""
    w, b = fold_bn(w, b, bn)
    co = w.shape[0]
    wp = w.permute(0, 2, 3, 1)                               # [co, kh, kw, ci]
    if pad_in > wp.shape[3]:
        wp = torch.cat([wp, wp.new_zeros(*wp.shape[:3], pad_in - wp.shape[3])], dim=3)
    wg = wp.reshape(co, -1)
    if pad_out > co:
        wg = torch.cat([wg, wg.new_zeros(pad_out - co, wg.shape[1])])
        b = torch.cat([b, b.new_zeros(pad_out - co)])
    return wg.to(torch.bfloat16).contiguous(), b.contiguous()


def prep_convT(w: torch.Tensor, b: torch.Tensor):
    """ConvTranspose2d [Cin, Cout, 2, 2] -> 4 per-tap bf16 [Cout, Cin] matrices + fp32 bias."""
    w = w.detach().float()
    taps = [w[:, :, t >> 1, t & 1].t().contiguous().to(torch.bfloat16) for t in range(4)]
    return taps, b.detach().float().contiguous()


_TAP_MAPS: dict = {}


def tap_maps(B: int, H: int, W: int, device) -> list:
    """int32 destination rows of the 4 taps of a k2 s2 transposed conv on a [B, H, W] grid."""
    key = (B, H, W, str(device))
    if key not in _TAP_MAPS:
        b = torch.arange(B, device=device).view(B, 1, 1)
        y = torch.arange(H, device=device).view(1, H, 1)
        x = torch.arange(W, device=device).view(1, 1, W)
        maps = []
        for t in range(4):
            ty, tx = t >> 1, t & 1
            dst = (b * 2 * H + 2 * y + ty) * (2 * W) + 2 * x + tx
            maps.append(dst.reshape(-1).to(torch.int32).contiguous())
        _TAP_MAPS[key] = maps
    return _TAP_MAPS[key]


# ------------------------------------------------------------------------------ conv helpers (NHWC bf16)
def conv1x1(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, act=None, residual=None,
            out_dtype=torch.bfloat16) -> torch.Tensor:
    B, H, W, C = x.shape
    res = residual.reshape(B * H * W, -1) if residual is not None else None
    y = _lib.gemm(x.reshape(B * H * W, C), w, b, act=act, residual=res, out_dtype=out_dtype)
    return y.view(B, H, W, -1)


def conv3x3(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, act=None, residual=None, stride: int = 1,
            out_dtype=torch.bfloat16) -> torch.Tensor:
    B, H, W, C = x.shape
    if stride == 1 and _lib.conv3x3_ok(B, H, W, C):      # implicit GEMM: no im2col matrix
        res = residual.reshape(B * H * W, -1) if residual is not None else None
        return _lib.conv3x3_nhwc(x.contiguous(), w, b, act=act, residual=res, out_dtype=out_dtype).view(B, H, W, -1)
    col = _lib.im2col_nhwc(x, 3, 3, stride, 1)
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    res = residual.reshape(B * Ho * Wo, -1) if residual is not None else None
    y = _lib.gemm(col, w, b, act=act, residual=res, out_dtype=out_dtype)
    return y.view(B, Ho, Wo, -1)


def convT2x2(x: torch.Tensor, taps: list, b: torch.Tensor, act=None) -> torch.Tensor:
    B, H, W, C = x.shape
    co = taps[0].shape[0]
    out = torch.empty(B * 2 * H * 2 * W, co, device=x.device, dtype=torch.bfloat16)
    rows = x.reshape(B * H * W, C)
    for t, rm in enumerate(tap_maps(B, H, W, x.device)):
        _lib.gemm(rows, taps[t], b, out=out, row_map=rm, act=act)
    return out.view(B, 2 * H, 2 * W, co)


def ln_rows(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-6, gelu: bool = False,
            out_dtype=torch.bfloat16) -> torch.Tensor:
    B, H, W, C = x.shape
    return _lib.layernorm(x.reshape(B * H * W, C), w, b, eps, gelu=gelu, out_dtype=out_dtype).view(B, H, W, C)


def to_nhwc_bf16(x: torch.Tensor) -> torch.Tensor:
    """NCHW (any float dtype) -> NHWC bf16 (API-boundary conversion only)."""
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def to_nchw_f32(x: torch.Tensor) -> torch.Tensor:
    return _lib.nhwc_to_nchw(x.contiguous())


class _PrepMixin:
    def _init_prep(self):
        self._prep = None
        self.register_load_state_dict_post_hook(lambda *_: setattr(self, "_prep", None))

    def _apply(self, fn, *a, **k):
        self._prep = None
        return super()._apply(fn, *a, **k)


# ------------------------------------------------------------------------------ aggregators
def _seq(*mods) -> nn.Sequential:
    return nn.Sequential(*mods)


@MODELS.register_module(force=True)
class RSFeatureAggregator(_PrepMixin, BaseModule):
    """M:987-1057."""
    in_channels_dict = {"base": [768] * 13, "large": [1024] * 25, "huge": [1280] * 33}

    def __init__(self, in_channels, hidden_channels=64, out_channels=256, select_layers=range(1, 12, 2),
                 init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        assert isinstance(in_channels, str)
        arch = "base" if "base" in in_channels else "large" if "large" in in_channels else "huge"
        self.in_channels = self.in_channels_dict[arch]
        self.select_layers = list(select_layers)
        hc, oc = hidden_channels, out_channels
        self.downconvs = nn.ModuleList(
            _seq(_conv(hc, self.in_channels[i], 1), _BN(hc), _Slot(), _conv(hc, hc, 3), _BN(hc), _Slot())
            for i in self.select_layers)
        self.hidden_convs = nn.ModuleList(_seq(_conv(hc, hc, 3), _BN(hc), _Slot()) for _ in self.select_layers)
        self.fusion_conv = _seq(_conv(oc, hc, 1), _BN(oc), _Slot(), _conv(oc, oc, 3), _BN(oc), _Slot(),
                                _conv(oc, oc, 3))
        self._init_prep()

    @torch.no_grad()
    def _prepare(self):
        # the 32 hidden channels ride in 64-channel maps (upper half exactly zero): 64 bf16 = one 128-byte swizzle atom,
        # so the 3x3 convs take the implicit-GEMM path (4-D TMA taps) instead of im2col + GEMM
        hc = self.downconvs[0][3].weight.shape[0]
        hp = (hc + 63) // 64 * 64
        p = {"down": [], "hid": []}
        for d in self.downconvs:
            p["down"].append((prep_conv(d[0].weight, d[0].bias, d[1], pad_out=hp),
                              prep_conv(d[3].weight, d[3].bias, d[4], pad_out=hp, pad_in=hp)))
        for h in self.hidden_convs:
            p["hid"].append(prep_conv(h[0].weight, h[0].bias, h[1], pad_out=hp, pad_in=hp))
        f = self.fusion_conv
        p["fus"] = (prep_conv(f[0].weight, f[0].bias, f[1], pad_in=hp), prep_conv(f[3].weight, f[3].bias, f[4]),
                    prep_conv(f[6].weight, f[6].bias, None))
        self._prep = p
        return p

    @torch.no_grad()
    def forward_nhwc(self, hidden_states) -> torch.Tensor:
        """hidden_states: L+1 fp32 NHWC maps (the encoder's output tuple) -> bf16 NHWC [B,h,w,out]."""
        assert len(hidden_states) == len(self.in_channels)
        p = self._prep or self._prepare()
        x = None
        for idx, il in enumerate(self.select_layers):
            hs = hidden_states[il]
            hb = _lib.cast_bf16(hs.contiguous()) if hs.dtype == torch.float32 else hs
            (w1, b1), (w2, b2) = p["down"][idx]
            f = conv1x1(hb, w1, b1, act="relu")
            # features[idx] (+ running x, M:1052-1053): ReLU first, then the residual
            hstate = conv3x3(f, w2, b2, act="relu", residual=x)
            wh, bh = p["hid"][idx]
            x = conv3x3(hstate, wh, bh, act="relu", residual=hstate)        # x = hidden + residual (M:1054-1055)
        (w1, b1), (w2, b2), (w3, b3) = p["fus"]
        x = conv1x1(x, w1, b1, act="relu")
        x = conv3x3(x, w2, b2, act="relu")
        return conv3x3(x, w3, b3)

    def forward(self, inputs):
        return to_nchw_f32(self.forward_nhwc([h for h in inputs]))


@MODELS.register_module(force=True)
class PseudoFeatureAggregator(_PrepMixin, BaseModule):
    """M:943-984: conv1x1 -> LN -> conv3x3 -> LN -> conv3x3 -> LN (all bias-free)."""

    def __init__(self, in_channels, hidden_channels=64, out_channels=256, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        hc, oc = hidden_channels, out_channels
        self.channel_fusion = _seq(_conv(hc, in_channels, 1, bias=False), _Affine((hc,)),
                                   _conv(hc, hc, 3, bias=False), _Affine((hc,)),
                                   _conv(oc, hc, 3, bias=False), _Affine((oc,)))
        self._init_prep()

    @torch.no_grad()
    def _prepare(self):
        c = self.channel_fusion
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        self._prep = dict(w=[prep_conv(c[i].weight, None)[0] for i in (0, 2, 4)],
                          ln=[(f32(c[i].weight), f32(c[i].bias)) for i in (1, 3, 5)])
        return self._prep

    @torch.no_grad()
    def forward_nhwc(self, x: torch.Tensor) -> torch.Tensor:
        p = self._prep or self._prepare()
        x = ln_rows(conv1x1(x, p["w"][0], None), *p["ln"][0])
        x = ln_rows(conv3x3(x, p["w"][1], None), *p["ln"][1])
        return ln_rows(conv3x3(x, p["w"][2], None), *p["ln"][2])

    def forward(self, inputs):
        assert len(inputs) == 1
        return to_nchw_f32(self.forward_nhwc(to_nhwc_bf16(inputs[0])))


class _ConvModule(nn.Module):
    """mmcv ConvModule(norm_cfg=LN2d, act_cfg=None): bias-free conv + LN2d (SURVEY 8c)."""

    def __init__(self, cin: int, cout: int, k: int):
        super().__init__()
        self.conv = _conv(cout, cin, k, bias=False)
        self.ln = _Affine((cout,))

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # mmcv names the norm after infer_abbr(LN2d) = 'norm_layer'; accept either spelling
        for suf in ("weight", "bias"):
            alt = f"{prefix}norm_layer.{suf}"
            if alt in state_dict and f"{prefix}ln.{suf}" not in state_dict:
                state_dict[f"{prefix}ln.{suf}"] = state_dict.pop(alt)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


@MODELS.register_module(force=True)
class RSSimpleFPN(_PrepMixin, BaseModule):
    """M:1277-1363 with norm_cfg=dict(type='LN2d')."""

    def __init__(self, backbone_channel, in_channels, out_channels, num_outs, conv_cfg=None, norm_cfg=None,
                 act_cfg=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        assert isinstance(in_channels, list) and len(in_channels) == 4
        assert norm_cfg is not None and norm_cfg.get("type") == "LN2d", "RSSimpleFPN is built with LN2d"
        bc = backbone_channel
        self.backbone_channel, self.in_channels = bc, in_channels
        self.out_channels, self.num_ins, self.num_outs = out_channels, 4, num_outs
        self.fpn1 = _seq(_ConvT(bc, bc // 2), _Affine((bc // 2,)), _Slot(), _ConvT(bc // 2, bc // 4))
        self.fpn2 = _seq(_ConvT(bc, bc // 2))
        self.fpn3 = _seq(_Slot())
        self.fpn4 = _seq(_Slot())
        self.lateral_convs = nn.ModuleList(_ConvModule(c, out_channels, 1) for c in in_channels)
        self.fpn_convs = nn.ModuleList(_ConvModule(out_channels, out_channels, 3) for _ in in_channels)
        self._init_prep()

    @torch.no_grad()
    def _prepare(self):
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        p = dict(t1a=prep_convT(self.fpn1[0].weight, self.fpn1[0].bias),
                 ln1=(f32(self.fpn1[1].weight), f32(self.fpn1[1].bias)),
                 t1b=prep_convT(self.fpn1[3].weight, self.fpn1[3].bias),
                 t2=prep_convT(self.fpn2[0].weight, self.fpn2[0].bias), lat=[], out=[])
        for l, o in zip(self.lateral_convs, self.fpn_convs):
            p["lat"].append((prep_conv(l.conv.weight, None)[0], f32(l.ln.weight), f32(l.ln.bias)))
            p["out"].append((prep_conv(o.conv.weight, None)[0], f32(o.ln.weight), f32(o.ln.bias)))
        self._prep = p
        return p

    @torch.no_grad()
    def forward_nhwc(self, x: torch.Tensor) -> list:
        p = self._prep or self._prepare()
        f1 = convT2x2(x, *p["t1a"])
        f1 = ln_rows(f1, *p["ln1"], gelu=True)
        f1 = convT2x2(f1, *p["t1b"])
        f2 = convT2x2(x, *p["t2"])
        f4 = _lib.pool2_nhwc(x, 0)
        outs = []
        for i, f in enumerate([f1, f2, x, f4]):
            wl, gl, bl = p["lat"][i]
            lat = ln_rows(conv1x1(f, wl, None), gl, bl)
            wo, go, bo = p["out"][i]
            outs.append(ln_rows(conv3x3(lat, wo, None), go, bo))
        for _ in range(self.num_outs - 4):
            outs.append(_lib.pool2_nhwc(outs[-1], 1))
        return outs

    def forward(self, input):
        return tuple(to_nchw_f32(o) for o in self.forward_nhwc(to_nhwc_bf16(input)))


@MODELS.register_module(force=True)
class RSFPN(BaseModule):
    """M:917-940."""

    def __init__(self, feature_aggregator=None, feature_spliter=None, init_cfg=None):
        BaseModule.__init__(self, init_cfg=None)
        if feature_aggregator is not None:
            self.feature_aggregator = MODELS.build(feature_aggregator)
        if feature_spliter is not None:
            self.feature_spliter = MODELS.build(feature_spliter)

    @torch.no_grad()
    def forward_nhwc(self, hidden_states, emb_nhwc: torch.Tensor | None = None) -> list:
        """hidden_states: the encoder's tuple (HF variant) or None with emb_nhwc (mmpretrain variant)."""
        if hasattr(self, "feature_aggregator"):
            agg = self.feature_aggregator
            if isinstance(agg, PseudoFeatureAggregator):
                x = agg.forward_nhwc(emb_nhwc)
            else:
                x = agg.forward_nhwc(hidden_states)
        else:
            x = emb_nhwc
        if hasattr(self, "feature_spliter"):
            return self.feature_spliter.forward_nhwc(x)
        return [x]

    def forward(self, inputs):
        x = self.feature_aggregator(inputs) if hasattr(self, "feature_aggregator") else inputs
        return self.feature_spliter(x) if hasattr(self, "feature_spliter") else (x,)


__all__ = ["LN2d", "RSFeatureAggregator", "PseudoFeatureAggregator", "RSSimpleFPN", "RSFPN"]
