"""Float64 restatements of the query head's standalone kernels (include/rsp_b200.h).  TEST INFRASTRUCTURE ONLY.

  * ``ms_deform_core``: rsp_ms_deform_attn_sample, the core of mmcv MultiScaleDeformableAttention without its
    projections (the core of restate_query.ms_deform_attn);
  * ``grouped_gemm``: rsp_gemm_bf16_grouped, one [N, K] weight per group of A rows, rows scattered by a map;
  * ``sam_mask_embed_src``: rsp_mask_embed_src, HF SamMaskEmbedding (restate.sam_mask_embedding run in float64) plus
    the image embedding of each prompt's image, and the key positional encoding for ``src_pe``.

Each ``*_tol`` bounds |kernel - reference| element by element from the kernel's rounding points, in the terms of
oracle/decoder_kernels.py: a bf16 result costs U8 |x|, an fp32 sum of K terms about K U24 sum|terms|.  The references
take the tensors the kernels read (bf16 or fp32) and compute in float64 on their device."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import restate
from .decoder_kernels import D, U8, U24, GELU_LIP, _ln_err

HEADS = 8


# ---------------------------------------------------------------------------------------------------- MSDeformAttn
def level_starts(shapes) -> list:
    s, out = 0, []
    for h, w in shapes:
        out.append(s)
        s += h * w
    return out


def deform_ref_points(shapes, level_of=None) -> torch.Tensor:
    """[NQ, 2] (x, y): the centre of each query's own cell, normalised by its level's (W, H).  level_of(l) names the
    level whose grid a query of level l is placed on (a defect when it is not l)."""
    refs = []
    for l, (h, w) in enumerate(shapes):
        hh, ww = shapes[l if level_of is None else level_of(l)]
        q = torch.arange(h * w, dtype=D)
        refs.append(torch.stack([(q % ww + 0.5) / ww, (torch.div(q, ww, rounding_mode="floor") + 0.5) / hh], dim=-1))
    return torch.cat(refs)


def _deform_split(ow: torch.Tensor, B: int, NQ: int, L: int, P: int):
    """ow [B NQ, >= 8 L P 3] as the kernel reads it -> offsets [B, NQ, 8, L, P, 2], logits [B, NQ, 8, L P]."""
    ow = ow.to(D)
    off = ow[:, :HEADS * L * P * 2].reshape(B, NQ, HEADS, L, P, 2)
    logit = ow[:, HEADS * L * P * 2:HEADS * L * P * 3].reshape(B, NQ, HEADS, L * P)
    return off, logit


def ms_deform_core(value: torch.Tensor, ow: torch.Tensor, shapes, points: int, *, norm=None, ref=None,
                   starts=None) -> torch.Tensor:
    """rsp_ms_deform_attn_sample: value [B, NQ, 8 hd] (the levels' pixels in order, each row-major), ow [B NQ, >= 8 L P
    3] = offsets (heads, levels, points, (x, y)) then logits (heads, levels points) -> [B NQ, 8 hd] float64.

    Sampling location = reference point (the centre of the query's own cell, for every level) + offset / (W_l, H_l);
    bilinear sampling of each level with zero padding (grid_sample, align_corners=False); weights = softmax over the
    L P logits of the head.  norm / ref / starts replace the normalisers [(nx, ny)], reference points or level starts
    (the CPU tests restate defects with them)."""
    B, NQ, E = value.shape
    hd, L, P = E // HEADS, len(shapes), points
    dev = value.device
    off, logit = _deform_split(ow, B, NQ, L, P)
    aw = torch.softmax(logit, dim=-1).view(B, NQ, HEADS, L, P)
    norm = torch.tensor([[w, h] for h, w in shapes] if norm is None else norm, dtype=D, device=dev)
    ref = (deform_ref_points(shapes) if ref is None else ref).to(dev)
    grids = 2 * (ref[None, :, None, None, None, :] + off / norm[None, None, None, :, None, :]) - 1
    starts = level_starts(shapes) if starts is None else starts
    vpad = torch.cat([value.to(D), value.new_zeros(B, max(h * w for h, w in shapes), E).to(D)], dim=1)
    out = torch.zeros(B, HEADS, hd, NQ, dtype=D, device=dev)
    for l, (h, w) in enumerate(shapes):
        v = vpad[:, starts[l]:starts[l] + h * w].reshape(B, h, w, HEADS, hd).permute(0, 3, 4, 1, 2)
        g = grids[:, :, :, l].transpose(1, 2).reshape(B * HEADS, NQ, P, 2)
        s = F.grid_sample(v.reshape(B * HEADS, hd, h, w), g, mode="bilinear", padding_mode="zeros",
                          align_corners=False)                                           # [B 8, hd, NQ, P]
        wl = aw[:, :, :, l].permute(0, 2, 1, 3).reshape(B * HEADS, 1, NQ, P)
        out += (s * wl).sum(-1).view(B, HEADS, hd, NQ)
    return out.permute(0, 3, 1, 2).reshape(B * NQ, E)


def ms_deform_tol(value: torch.Tensor, ow: torch.Tensor, shapes, points: int, ref: torch.Tensor) -> torch.Tensor:
    """Bound on |kernel - ms_deform_core|, [B NQ, 8 hd].  Per (query, head), with V = max |value| of the head:
      * sample position: the kernel forms x = (rx + off / W) W - 0.5 in fp32, within dx = 4 U24 (W + |off| + 1) of
        the exact position (y alike).  Bilinear sampling with zero padding is continuous, with slope <= 2 V along
        each axis, so a sample moves by <= 2 V (dx + dy) times its weight;
      * weights: logit - max, expf (2 ulp), a sum of L P terms and a division: relative error
        <= (|logit - max| + L P + 10) U24;
      * the fp32 sum of 4 L P weighted corners: (4 L P + 8) U24 V;
      * the bf16 output: U8 |ref|."""
    B, NQ, E = value.shape
    hd, L, P = E // HEADS, len(shapes), points
    off, logit = _deform_split(ow, B, NQ, L, P)
    aw = torch.softmax(logit, dim=-1).view(B, NQ, HEADS, L, P)
    d = (logit - logit.amax(-1, keepdim=True)).abs().view(B, NQ, HEADS, L, P)
    wh = torch.tensor([[w, h] for h, w in shapes], dtype=D, device=aw.device)             # [L, 2] (W, H)
    dpos = 4 * U24 * (wh[None, None, None, :, None, :] + off.abs() + 1)                     # [B, NQ, 8, L, P, 2]
    vmax = value.abs().to(D).reshape(B, NQ, HEADS, hd).amax(dim=(1, 3)).view(B, 1, HEADS)
    per = aw * (2 * dpos.sum(-1) + (d + L * P + 10) * U24)
    head = (per.sum(dim=(3, 4)) + (4 * L * P + 8) * U24) * vmax + 1e-30                    # [B, NQ, 8]
    head = head.repeat_interleave(hd, dim=-1).reshape(B * NQ, E)
    return head * (1 + U8) + U8 * ref.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------- grouped GEMM
def grouped_gemm(a: torch.Tensor, w: torch.Tensor, N: int, m_group_rows: int, w_group_rows: int,
                 row_map: torch.Tensor | None = None, out_rows: int | None = None, w_of_col=None) -> torch.Tensor:
    """rsp_gemm_bf16_grouped: out[row_map[m], n] = sum_k a[m, k] w[g w_group_rows + n, k], g = m // m_group_rows;
    rows with row_map -1 are not written.  -> float64 [out_rows, N], NaN where no row lands.  w_of_col(g, n) names
    the weight row a column reads (a defect when it is not g w_group_rows + n); rows past w read as 0."""
    M = a.shape[0]
    out = torch.full((M if out_rows is None else out_rows, N), float("nan"), dtype=D, device=a.device)
    wz = torch.cat([w.to(D), w.new_zeros(N + w_group_rows, w.shape[1]).to(D)])
    cols = torch.arange(N, device=a.device)
    for g in range(M // m_group_rows):
        rows = torch.arange(g * m_group_rows, (g + 1) * m_group_rows, device=a.device)
        wr = g * w_group_rows + cols if w_of_col is None else w_of_col(g, cols)
        res = a[rows].to(D) @ wz[wr].t()
        dst = rows if row_map is None else row_map[rows].long()
        keep = dst >= 0
        out[dst[keep]] = res[keep]
    return out


def grouped_gemm_tol(a: torch.Tensor, w: torch.Tensor, N: int, m_group_rows: int, w_group_rows: int, ref,
                     row_map: torch.Tensor | None = None, out_bf16: bool = False) -> torch.Tensor:
    """K U24 sum_k |a| |w| (the fp32 accumulator) + the output rounding (bf16: U8 |ref|, fp32: U24 |ref|)."""
    mag = grouped_gemm(a.abs(), w.abs(), N, m_group_rows, w_group_rows, row_map, ref.shape[0])
    return a.shape[1] * U24 * mag + (U8 if out_bf16 else U24) * ref.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------- mask embedding
def mask_embed_sd(weights: list) -> dict:
    """The 10 kernel weights (conv1 w, b, ln1 g, b, conv2 w, b, ln2 g, b, conv3 w [256, 16], b) as the float64 state
    dict of restate.sam_mask_embedding."""
    names = ["conv1.weight", "conv1.bias", "layer_norm1.weight", "layer_norm1.bias", "conv2.weight", "conv2.bias",
             "layer_norm2.weight", "layer_norm2.bias", "conv3.weight", "conv3.bias"]
    sd = {"mask_embed." + k: t.to(D) for k, t in zip(names, weights)}
    sd["mask_embed.conv3.weight"] = sd["mask_embed.conv3.weight"].reshape(-1, 16, 1, 1)
    return sd


def _rows(x: torch.Tensor) -> torch.Tensor:
    """NCHW -> channels-last rows [N h w, C]."""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def sam_mask_embed_src(mpp: torch.Tensor, weights: list, emb: torch.Tensor, pos: torch.Tensor, n_per_img: int,
                       hw: tuple, eps: float = 1e-6):
    """rsp_mask_embed_src: mpp fp32 [N, 4h, 4w] mask logits, emb [images, h w, 256] image embedding rows, pos [h w, 256]
    -> (src, src_pe) float64 [N h w, 256]: SamMaskEmbedding(mpp[n]) + emb[n // n_per_img], and that + pos."""
    N = mpp.shape[0]
    h, w = hw
    dense = _rows(restate.sam_mask_embedding(mask_embed_sd(weights), mpp.to(D).unsqueeze(1), eps))
    img = torch.arange(N, device=mpp.device) // n_per_img
    src = dense + emb.to(D)[img].reshape(N * h * w, 256)
    return src, src + pos.to(D).repeat(N, 1)


def _gelu_eval(y: torch.Tensor) -> torch.Tensor:
    """fp32 0.5 x (1 + erff(x / sqrt 2)): erff within 2 ulp of 1, then three roundings."""
    return 4 * U24 * (y.abs() + F.gelu(y).abs())


def _ln_cf_err(x: torch.Tensor, dx: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float):
    """(LN output, error bound) of a channels-first LayerNorm over the C of NCHW x carrying dx: decoder_kernels._ln_err
    plus rsqrtf (2 ulp) and the affine's roundings."""
    xr, dr = x.permute(0, 2, 3, 1), dx.permute(0, 2, 3, 1)
    y = F.layer_norm(xr, (xr.shape[-1],), g.to(D), b.to(D), eps)
    e = _ln_err(xr, dr, g, eps) + 4 * U24 * (y.abs() + b.to(D).abs())
    return y.permute(0, 3, 1, 2), e.permute(0, 3, 1, 2)


def mask_embed_src_tol(mpp: torch.Tensor, weights: list, src_ref: torch.Tensor, mma: bool, eps: float = 1e-6,
                       pos: torch.Tensor | None = None) -> torch.Tensor:
    """Bound on |kernel - sam_mask_embed_src|, [N h w, 256], carried stage by stage through the fp32 kernel's
    arithmetic: each conv is an fp32 sum (K + 2) U24 sum|terms| plus its inputs' errors times |weights|; each LayerNorm
    goes through decoder_kernels._ln_err; each GELU is GELU_LIP-Lipschitz and evaluated within _gelu_eval.  The mma
    kernel (mma=True) also rounds the hidden vector and conv3's weight to bf16: U8 |h| and |w3 - bf16(w3)|.  Then the
    embedding add, and the bf16 output rounding U8 |ref|.  pos: the bound of src_pe = src + pos instead."""
    w1, b1, g1, be1, w2, b2, g2, be2, w3, b3 = [t.to(D) for t in weights]
    m = mpp.to(D).unsqueeze(1)
    x1 = F.conv2d(m, w1, b1, stride=2)
    dx1 = 6 * U24 * (F.conv2d(m.abs(), w1.abs(), b1.abs(), stride=2))
    y1, e1 = _ln_cf_err(x1, dx1, g1, be1, eps)
    h1 = F.gelu(y1)
    dh1 = GELU_LIP * e1 + _gelu_eval(y1)
    x2 = F.conv2d(h1, w2, b2, stride=2)
    dx2 = F.conv2d(dh1, w2.abs(), stride=2) + 18 * U24 * F.conv2d(h1.abs(), w2.abs(), b2.abs(), stride=2)
    y2, e2 = _ln_cf_err(x2, dx2, g2, be2, eps)
    h2 = _rows(F.gelu(y2))
    dh2 = _rows(GELU_LIP * e2 + _gelu_eval(y2))
    w3a = w3.reshape(256, 16).abs()
    mag = h2.abs() @ w3a.t()
    dout = dh2 @ w3a.t() + 18 * U24 * (mag + b3.abs())
    if mma:      # bf16 hidden vector: U8 |h| (on h and on its error); bf16 w3: exactly |w3 - bf16(w3)|
        w3r = (w3.reshape(256, 16) - w3.reshape(256, 16).to(torch.bfloat16).to(D)).abs()
        dout = dout + U8 * (dh2 @ w3a.t()) + U8 * mag + h2.abs() @ w3r.t()
    ref = src_ref if pos is None else src_ref - pos.to(D).repeat(src_ref.shape[0] // pos.shape[0], 1)
    dout = dout + 2 * U24 * (ref.abs() + src_ref.abs())
    return dout * (1 + U8) + U8 * src_ref.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------- input builders
def deform_inputs(shapes, points: int, hd: int, B: int, seed: int, logits: str = "normal"):
    """value bf16 [B, NQ, 8 hd] with per-head offsets; ow fp32 [B NQ, 8 L P 3] (+ 5 unread columns, so ld_ow > the
    row) whose offsets put the samples, cycling over the points:
      fully outside the map (|off| >= size + 2), half outside (one to three corners past an edge), on integer and
      half-integer pixel positions, exactly at x = -1 and x = W (y likewise), and anywhere inside.
    logits: "normal" (N(0, 2)), "spread" (spreads above 80: the softmax must subtract the max), "equal" (all 0)."""
    g = torch.Generator().manual_seed(seed)
    L, P = len(shapes), points
    NQ = sum(h * w for h, w in shapes)
    value = torch.randn(B, NQ, HEADS, hd, generator=g) + (2.0 * torch.arange(HEADS) - 7.0).view(1, 1, HEADS, 1)
    value = value.reshape(B, NQ, HEADS * hd).to(torch.bfloat16)
    ref = deform_ref_points(shapes).float()                                     # [NQ, 2] (x, y) normalised
    wh = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32)         # [L, 2]
    off = torch.empty(B, NQ, HEADS, L, P, 2)
    for l in range(L):
        pix_ref = ref[:, None, None, :] * wh[l] - 0.5                            # [NQ, 1, 1, 2] ref in pixels of l
        for p in range(P):
            kind = (p + l) % 5
            u = torch.rand(B, NQ, HEADS, 2, generator=g)
            sgn = torch.where(torch.rand(B, NQ, HEADS, 2, generator=g) < 0.5, -1.0, 1.0)
            if kind == 0:      # anywhere inside
                target = u * (wh[l] - 1)
            elif kind == 1:    # fully outside: 1.5 .. 3 pixels past an edge, or far away
                target = torch.where(sgn < 0, -2.5 - 3 * u, wh[l] + 1.5 + 3 * u)
            elif kind == 2:    # half outside: within one pixel past an edge (1 to 3 corners dropped)
                target = torch.where(sgn < 0, -u, wh[l] - 1 + u)
            elif kind == 3:    # integer and half-integer pixel positions
                target = torch.floor(u * wh[l] * 2) / 2 - 0.5 * (torch.rand(B, NQ, HEADS, 2, generator=g) < 0.3)
            else:              # exactly x = -1 or x = W: the one in-map tap has weight 0
                target = torch.where(sgn < 0, torch.full_like(u, -1.0), wh[l].expand_as(u))
            off[:, :, :, l, p] = target - pix_ref.view(1, NQ, 1, 2)
    if logits == "spread":
        lg = 30 * torch.randn(B, NQ, HEADS, L * P, generator=g)
        lg[..., 0] = lg[..., 0] + 90                                            # spread > 80 in every row
    elif logits == "equal":
        lg = torch.full((B, NQ, HEADS, L * P), 3.25)
    else:
        lg = 2 * torch.randn(B, NQ, HEADS, L * P, generator=g)
    ow = torch.cat([off.reshape(B * NQ, -1), lg.reshape(B * NQ, -1), torch.randn(B * NQ, 5, generator=g)], dim=1)
    return value, ow.float()


def grouped_inputs(B: int, nq: int, hw_l: int, seed: int, C: int = 256):
    """The query head's call: me_pad bf16 [B 128, C] (rows 128 b + q, q < nq, hold image b's mask embeddings; the 28
    padding rows are not 0 here, so a padding row written anywhere shows), mf bf16 [B hw_l, C] (image b's resized
    mask features, exactly B hw_l rows: the last group has no slack), back int32 [B 128] (padded row -> compact
    row b nq + q, -1 on padding).  Image b's features are scaled by 10^(b % 4 - 1), so columns computed with another
    group's weights are off by orders of magnitude."""
    g = torch.Generator().manual_seed(seed)
    me = torch.randn(B * 128, C, generator=g).to(torch.bfloat16)
    scale = (10.0 ** (torch.arange(B) % 4 - 1.0)).repeat_interleave(hw_l).view(-1, 1)
    mf = (torch.randn(B * hw_l, C, generator=g) * 0.1 * scale).to(torch.bfloat16)
    back = torch.full((B, 128), -1, dtype=torch.int32)
    back[:, :nq] = (torch.arange(B).view(B, 1) * nq + torch.arange(nq).view(1, nq)).int()
    return me, mf, back.reshape(-1)


def mask_embed_weights(seed: int, bf16_w3: bool = True) -> list:
    """Weights for rsp_mask_embed_src in the kernel's layout.  ln2 puts channels 0-7 at pre-activations -3.9 .. -3.1,
    where erf and tanh GELU differ by 15 - 45 % of the value, and conv3's rows 0-127 read only those channels, so a
    GELU defect shows against the bf16 output rounding; rows 128-255 read all 16 channels."""
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randn(4, 1, 2, 2, generator=g) * 0.5
    b1 = 0.1 * torch.randn(4, generator=g)
    g1, be1 = 1 + 0.2 * torch.randn(4, generator=g), 0.2 * torch.randn(4, generator=g)
    w2 = torch.randn(16, 4, 2, 2, generator=g) * 0.25
    b2 = 0.1 * torch.randn(16, generator=g)
    g2, be2 = 1 + 0.2 * torch.randn(16, generator=g), 0.3 * torch.randn(16, generator=g)
    g2[:8], be2[:8] = 0.1 * (1 + 0.1 * torch.rand(8, generator=g)), -3.5
    w3 = 0.25 * torch.randn(256, 16, generator=g)
    w3[:128, 8:] = 0
    w3[:128, :8] = w3[:128, :8].abs()
    if bf16_w3:
        w3 = w3.to(torch.bfloat16).float()
    b3 = 0.1 * torch.randn(256, generator=g)
    b3[:128] = 0
    return [t.float().contiguous() for t in (w1, b1, g1, be1, w2, b2, g2, be2, w3, b3)]


def mask_embed_inputs(N: int, hw: tuple, n_per_img: int, seed: int):
    """mpp fp32 [N, 4h, 4w]: mask logits of magnitude up to 20, exact-zero 4 x 4 patches and constant 4 x 4 patches;
    emb fp32 [N / n_per_img, h w, 256] (image b's rows offset by 3 b, so the wrong image shows); pos fp32 [h w, 256]."""
    g = torch.Generator().manual_seed(seed)
    h, w = hw
    mpp = 20 * torch.tanh(torch.randn(N, 4 * h, 4 * w, generator=g))
    patch = torch.rand(N, h, w, generator=g)
    pv = torch.round(8 * torch.randn(N, h, w, generator=g)) / 2
    const = torch.where(patch < 0.15, torch.zeros_like(pv), pv).repeat_interleave(4, 1).repeat_interleave(4, 2)
    sel = (patch < 0.3).repeat_interleave(4, 1).repeat_interleave(4, 2)
    mpp = torch.where(sel, const, mpp).contiguous()
    n_img = N // n_per_img
    emb = torch.randn(n_img, h * w, 256, generator=g) * 0.5 + 3.0 * torch.arange(n_img).view(-1, 1, 1)
    emb[:, :, :128] = 0          # conv3's sensitive rows are compared without an offset
    pos = torch.randn(h * w, 256, generator=g)
    return mpp, emb.contiguous(), pos.contiguous()
