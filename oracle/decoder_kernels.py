"""Float64 restatements of the mask decoder's kernel contracts (include/rsp_b200.h).  TEST INFRASTRUCTURE ONLY.

One function per kernel entry point, written from the header and from HF's SamAttention (HF:231-270) and upscaler
(HF:515-531) arithmetic.  Each rounds to bf16 only where the header makes the kernel's intermediate bf16: the k | v
and Q projections of the fused kernels and the attention output that feeds i2t_fused's out_proj.  Everything else,
the softmax included, is float64.  The final output is returned unrounded: a test's tolerance includes the kernel's
own output rounding, which is a tighter comparison than two rounded values.

The weight layouts are those of ``SamMaskDecoderB200._prepare()``: ``convt_gemm_weight`` / ``convt_gemm_bias`` turn a
ConvTranspose2d(k=2, s=2) into a GEMM whose output columns are (tap = ty * 2 + tx, channel), and ``kvw`` is the
k_proj rows followed by the v_proj rows.

``*_tol`` give per-element bounds on |kernel - reference| from the kernel's rounding points:
  * a bf16 result costs U8 |x|, U8 = 2^-8 the unit roundoff of bf16 (8 significant bits);
  * bf16 probabilities P in P V cost <= U8 max|V| per head (the row sum l is taken on the unrounded P);
  * an fp32 sum of K terms costs about K U24 sum|terms|, U24 = 2^-24;
  * a logit error ds moves a softmax-weighted mean by <= 2 ds max|V|.
The builders make the adversarial inputs the CPU and GPU tests share.  Functions take tensors on any device and
compute in float64 there (the GPU tests run the large cases on the GPU)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

D = torch.float64
U8 = 2.0 ** -8
U24 = 2.0 ** -24
GELU_FAST_ERR = 4e-6      # sm90.cuh gelu_fast: |error| <= 3.6e-6 on [-9, 9], exact saturation beyond
GELU_LIP = 1.13           # max |GELU'(x)|
CHUNK = 64                # prompts per float64 block (bounds the [prompts, heads, Tq, HW] logits)


def rb(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest even), back to float64."""
    return x.to(torch.bfloat16).to(D)


def convt_gemm_weight(w: torch.Tensor) -> torch.Tensor:
    """ConvTranspose2d weight [cin, cout, 2, 2] -> GEMM weight [4 cout, cin], rows (tap = ty * 2 + tx, cout)."""
    return w.permute(2, 3, 1, 0).reshape(4 * w.shape[1], w.shape[0])


def convt_gemm_bias(b: torch.Tensor) -> torch.Tensor:
    return b.repeat(4)


def _rows(t: torch.Tensor, block: torch.Tensor | None, n: int, hw: int) -> torch.Tensor:
    """Rows blk * hw .. + hw of t for each prompt (blk = block[p], or p): [n, hw, C]."""
    blk = torch.arange(n, device=t.device) if block is None else block.to(t.device).long()
    return t.reshape(-1, hw, t.shape[-1])[blk]


def _core(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """softmax(q k^T / sqrt(c)) v per head, float64: q [n, Tq, heads c], k / v [n, Tk, heads c]."""
    n, tq, dm = q.shape
    c = dm // heads
    sp = lambda t: t.to(D).reshape(n, t.shape[1], heads, c).transpose(1, 2)  # noqa: E731
    s = (sp(q) @ sp(k).transpose(2, 3)) * c ** -0.5
    return (torch.softmax(s, dim=-1) @ sp(v)).transpose(1, 2).reshape(n, tq, dm)


def token_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """rsp_token_self_attention: q, k, v [N, T, heads c] -> [N, T, heads c]."""
    return _core(q, k, v, heads)


def t2i(q: torch.Tensor, K: torch.Tensor, V: torch.Tensor, hw: int, kv_block: torch.Tensor | None = None) -> torch.Tensor:
    """rsp_t2i_attention: q [N, Tq, 128] (8 heads x 16) attends to rows kv_block[n] * hw .. + hw of K, V [*, 128]."""
    n = q.shape[0]
    out = []
    for p0 in range(0, n, CHUNK):
        sl = slice(p0, min(n, p0 + CHUNK))
        blk = None if kv_block is None else kv_block[sl]
        if blk is None:
            blk = torch.arange(sl.start, sl.stop)
        out.append(_core(q[sl], _rows(K, blk, sl.stop - sl.start, hw), _rows(V, blk, sl.stop - sl.start, hw), 8))
    return torch.cat(out)


def i2t(Q: torch.Tensor, ktok: torch.Tensor, vtok: torch.Tensor, hw: int, q_block: torch.Tensor | None = None) -> torch.Tensor:
    """rsp_i2t_attention: rows q_block[n] * hw .. + hw of Q [*, 128] attend to ktok, vtok [N, Tq, 128] -> [N hw, 128]."""
    n = ktok.shape[0]
    out = []
    for p0 in range(0, n, CHUNK):
        sl = slice(p0, min(n, p0 + CHUNK))
        blk = torch.arange(sl.start, sl.stop) if q_block is None else q_block[sl]
        out.append(_core(_rows(Q, blk, sl.stop - sl.start, hw), ktok[sl], vtok[sl], 8).reshape(-1, 128))
    return torch.cat(out)


def t2i_fused(q, keys, kvw, kvb, pe_kv, hw: int) -> torch.Tensor:
    """rsp_t2i_fused: [K | V] = bf16((keys Wkv^T + kvb) + pe_kv[row % hw]), then t2i."""
    kv = rb(keys.to(D) @ kvw.to(D).t() + kvb.to(D) + pe_kv.to(D).repeat(keys.shape[0] // hw, 1))
    return t2i(q, kv[:, :128], kv[:, 128:], hw)


def i2t_fused(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln: tuple, hw: int) -> torch.Tensor:
    """rsp_i2t_fused: LN((bf16(i2t(Q)) Wo^T + ob) + keys) with Q = bf16((keys Wq^T + qb) + pe_q[row % hw])."""
    g, b, eps = ln
    Q = rb(keys.to(D) @ wq.to(D).t() + qb.to(D) + pe_q.to(D).repeat(keys.shape[0] // hw, 1))
    att = rb(i2t(Q, ktok, vtok, hw))
    return ln_row(att, wo, ob, keys, g, b, eps)


def _res_rows(residual, m: int, res_mod: int = 0, res_block_map=None, res_block_rows: int = 0) -> torch.Tensor:
    r = torch.arange(m, device=residual.device)
    if res_block_map is not None:
        r = res_block_map.to(residual.device).long()[r // res_block_rows] * res_block_rows + r % res_block_rows
    elif res_mod:
        r = r % res_mod
    return residual[r].to(D)


def ln_row(a, w, bias, residual, gamma, beta, eps: float, res_mod: int = 0, res_block_map=None,
           res_block_rows: int = 0) -> torch.Tensor:
    """rsp_gemm_bf16 epi_mode 1: LayerNorm_N(a W^T + bias + residual[rrow]) * gamma + beta, float64."""
    x = a.to(D) @ w.to(D).t()
    if bias is not None:
        x = x + bias.to(D)
    if residual is not None:
        x = x + _res_rows(residual, x.shape[0], res_mod, res_block_map, res_block_rows)
    return F.layer_norm(x, (x.shape[1],), gamma.to(D), beta.to(D), eps)


def up1_rows_to_image(rows: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """epi_mode 2 output rows [N h w, 4 * C] (pixel, (tap = ty * 2 + tx, C)) -> NCHW [N, C, 2h, 2w]."""
    c = rows.shape[1] // 4
    return rows.reshape(-1, h, w, 2, 2, c).permute(0, 5, 1, 3, 2, 4).reshape(-1, c, 2 * h, 2 * w)


def image_to_up1_rows(img: torch.Tensor) -> torch.Tensor:
    """NCHW [N, C, 2h, 2w] -> [N h w 4, C]: the epi_mode 3 operand, rows (prompt, y, x, tap1 = ty1 * 2 + tx1)."""
    n, c, h2, w2 = img.shape
    return img.reshape(n, c, h2 // 2, 2, w2 // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(-1, c)


def upscale1_ln_gelu(keys, up1_w, up1_b, gamma, beta, eps: float, h: int, w: int,
                     approximate: str = "none") -> torch.Tensor:
    """epi_mode 2: ConvTranspose2d(k2, s2) as keys up1_w^T + up1_b, LayerNorm over each tap's channels, erf GELU;
    keys [N h w, Cin] -> [N, C, 2h, 2w]."""
    y = keys.to(D) @ up1_w.to(D).t() + up1_b.to(D)
    c = y.shape[1] // 4
    y = F.layer_norm(y.view(-1, 4, c), (c,), gamma.to(D), beta.to(D), eps)
    return up1_rows_to_image(F.gelu(y, approximate=approximate).reshape(-1, 4 * c), h, w)


def upscale2_hyper(up1, up2_w, up2_b, hyper, h: int, w: int, approximate: str = "none") -> torch.Tensor:
    """epi_mode 3: mask[p, 4y + 2ty1 + ty2, 4x + 2tx1 + tx2] = sum_c GELU(up1 up2_w^T + up2_b)[(tap2, c)] hyper[p, c],
    up1 [P h w 4, Cin] rows (prompt, y, x, tap1) -> [P, 4h, 4w]."""
    P = hyper.shape[0]
    u = F.gelu(up1.to(D) @ up2_w.to(D).t() + up2_b.to(D), approximate=approximate)     # [P h w 4, (tap2, c)]
    c = hyper.shape[1]
    m = (u.view(P, h * w * 16, c) * hyper.to(D).view(P, 1, c)).sum(-1)
    return m.view(P, h, w, 2, 2, 2, 2).permute(0, 1, 3, 5, 2, 4, 6).reshape(P, 4 * h, 4 * w)


# ---------------------------------------------------------------------------------------------------- tolerances
def attention_tol(qabs1: torch.Tensor, kmax: torch.Tensor, vmax: torch.Tensor, c: int, tk: int, ref: torch.Tensor,
                  p_bf16: bool) -> torch.Tensor:
    """Bound on |kernel - ref| of an attention output, [rows, Tq, heads c] like ref.

    qabs1 [rows, Tq, heads] = scale * sum_c |q| of each query; kmax / vmax [rows, heads] = max |k| / |v| over the
    keys it attends to.  Terms: the logits are fp32 dot products of c terms, shifted by the row max and taken
    through __expf (ds <= (c + 12) U24 scale |q|_1 max|k| + 2^-21); P V and the row sum add tk terms in fp32; P is
    rounded to bf16 when p_bf16; the output is rounded to bf16."""
    ds = (c + 12) * U24 * qabs1 * kmax.unsqueeze(1) + 2.0 ** -21
    vm = vmax.unsqueeze(1)
    head = 2 * ds * vm + tk * U24 * vm + (U8 * vm if p_bf16 else 0)
    head = head.repeat_interleave(c, dim=-1)
    return head * (1 + U8) + (U8 + tk * U24) * ref.abs() + 1e-30


def _head_max(t: torch.Tensor, heads: int) -> torch.Tensor:
    """max |t| over all but the first dim and within each head's channels: [n, *, heads c] -> [n, heads]."""
    n = t.shape[0]
    return t.abs().to(D).reshape(n, -1, heads, t.shape[-1] // heads).amax(dim=(1, 3))


def _head_l1(t: torch.Tensor, heads: int) -> torch.Tensor:
    return t.abs().to(D).reshape(*t.shape[:-1], heads, t.shape[-1] // heads).sum(-1)


def token_attention_tol(q, k, v, heads: int, ref) -> torch.Tensor:
    c = q.shape[-1] // heads
    return attention_tol(_head_l1(q, heads) * c ** -0.5, _head_max(k, heads), _head_max(v, heads), c, q.shape[1],
                         ref, p_bf16=False)


def t2i_tol(q, K, V, hw: int, ref, kv_block=None) -> torch.Tensor:
    blk = torch.arange(q.shape[0]) if kv_block is None else kv_block.long().cpu()
    kmax = _head_max(K.reshape(-1, hw, 128), 8)[blk.to(K.device)]
    vmax = _head_max(V.reshape(-1, hw, 128), 8)[blk.to(V.device)]
    return attention_tol(_head_l1(q, 8) * 0.25, kmax, vmax, 16, hw, ref, p_bf16=True)


def i2t_tol(Q, ktok, vtok, hw: int, ref, q_block=None) -> torch.Tensor:
    n, tq = ktok.shape[:2]
    blk = torch.arange(n) if q_block is None else q_block.long().cpu()
    qabs1 = _head_l1(Q.reshape(-1, hw, 128), 8)[blk.to(Q.device)].reshape(n * hw, 1, 8) * 0.25
    kmax = _head_max(ktok, 8).repeat_interleave(hw, dim=0)
    vmax = _head_max(vtok, 8).repeat_interleave(hw, dim=0)
    return attention_tol(qabs1, kmax, vmax, 16, tq, ref.view(n * hw, 1, 128), p_bf16=True).view(n * hw, 128)


def _ln_err(x: torch.Tensor, dx: torch.Tensor, gamma: torch.Tensor, eps: float) -> torch.Tensor:
    """Bound on the error of LayerNorm over the last dim of x (fp32 statistics, shifted sums) when x carries dx:
    |d xhat_i| <= r (|dx_i| + max|dx| (1 + |xhat_i|)) plus 4 n U24 r max|x - mean| (1 + |xhat_i|)."""
    n = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    r = (x.var(-1, unbiased=False, keepdim=True) + eps).rsqrt()
    xhat = (x - mu) * r
    spread = (x - mu).abs().amax(-1, keepdim=True)
    dxm = dx.amax(-1, keepdim=True)
    return gamma.to(D).abs() * r * (dx + (dxm + 4 * n * U24 * spread) * (1 + xhat.abs()))


def ln_row_tol(a, w, bias, residual, gamma, beta, eps: float, ref, out_bf16: bool, **rmap) -> torch.Tensor:
    """Bound for ln_row: the accumulator is an fp32 sum of K products, then bias and residual are added in fp32."""
    K = a.shape[1]
    acc = a.to(D) @ w.to(D).t()
    x = acc + (0 if bias is None else bias.to(D))
    dx = K * U24 * (a.to(D).abs() @ w.to(D).abs().t())
    if residual is not None:
        x = x + _res_rows(residual, x.shape[0], **rmap)
    dx = dx + 3 * U24 * x.abs().amax(-1, keepdim=True)
    return _ln_err(x, dx, gamma, eps) + 3 * U24 * ref.abs() + (U8 if out_bf16 else U24) * ref.abs() + 1e-30


def upscale1_tol(keys, up1_w, up1_b, gamma, eps: float, h: int, w: int, ref) -> torch.Tensor:
    """Bound for upscale1_ln_gelu on the epi_mode 2 kernel: fp32 GEMM + LN, GELU within GELU_FAST_ERR, bf16 out."""
    K = keys.shape[1]
    x = keys.to(D) @ up1_w.to(D).t() + up1_b.to(D)
    dx = K * U24 * (keys.to(D).abs() @ up1_w.to(D).abs().t()) + 2 * U24 * x.abs()
    c = x.shape[1] // 4
    e = _ln_err(x.view(-1, 4, c), dx.view(-1, 4, c), gamma, eps).reshape(-1, 4 * c)
    e = GELU_LIP * e + GELU_FAST_ERR
    return up1_rows_to_image(e, h, w) * (1 + U8) + U8 * ref.abs() + 1e-30


def upscale2_tol(up1, up2_w, up2_b, hyper, h: int, w: int) -> torch.Tensor:
    """Bound for upscale2_hyper: fp32 GEMM over K, GELU within GELU_FAST_ERR, an fp32 sum of the 32 products."""
    P, c = hyper.shape
    K = up1.shape[1]
    x = up1.to(D) @ up2_w.to(D).t() + up2_b.to(D)
    dx = K * U24 * (up1.to(D).abs() @ up2_w.to(D).abs().t()) + 2 * U24 * x.abs()
    du = GELU_LIP * dx + GELU_FAST_ERR + 2 * U24 * F.gelu(x).abs()
    hy = hyper.to(D).abs().view(P, 1, c)
    e = (du.view(P, -1, c) * hy).sum(-1) + (c + 2) * U24 * (F.gelu(x).abs().view(P, -1, c) * hy).sum(-1)
    return e.view(P, h, w, 2, 2, 2, 2).permute(0, 1, 3, 5, 2, 4, 6).reshape(P, 4 * h, 4 * w) + 1e-30


def gelu_erf64(x: torch.Tensor) -> torch.Tensor:
    x = x.to(D)
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2.0)))


# ---------------------------------------------------------------------------------------------------- input builders
def _head_offsets(dev=None) -> torch.Tensor:
    """Per-head value offsets (-7 .. 7 in steps of 2), so output of a mixed-up head lands far from the right one."""
    return (2.0 * torch.arange(8, device=dev) - 7.0).repeat_interleave(16)


def token_inputs(n: int, t: int, heads: int, c: int, seed: int):
    """q, k, v bf16 [n, t, heads c] with sharp logits (|s| up to ~30) and per-head value offsets."""
    g = torch.Generator().manual_seed(seed)
    q = 2.5 * torch.randn(n, t, heads * c, generator=g)
    k = 2.5 * torch.randn(n, t, heads * c, generator=g)
    v = torch.randn(n, t, heads * c, generator=g) + 2.0 * torch.arange(heads).repeat_interleave(c) - heads
    return [x.to(torch.bfloat16) for x in (q, k, v)]


def t2i_inputs(n: int, hw: int, tq: int, blocks: int, seed: int, kv_block: list | None = None, shared: bool = False):
    """q [n, tq, 128], K, V [blocks hw, 128] bf16 (views of one [blocks hw, 256] matrix, row stride 256, when shared),
    kv_block int32 [n] (None: blocks == n, prompt n reads block n).

    Adversarial: in every block, the last key carries head h's sharpest logit for token h % tq (half of that token's
    softmax mass) and a distinct value (+12), so counting the clamped copies of that row a partial last tile stages
    past hw moves the output by several units; head h's values are offset by 2h - 7 and block b's by 3b, so reading
    another head or another block's rows shows."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n, tq, 128, generator=g)
    u = torch.randn(8, 16, generator=g)
    for h in range(8):
        q[:, h % tq, 16 * h:16 * h + 16] = u[h]
    q = q.to(torch.bfloat16)
    K = torch.randn(blocks, hw, 128, generator=g)
    V = torch.randn(blocks, hw, 128, generator=g) + _head_offsets() + 3.0 * torch.arange(blocks).view(-1, 1, 1)
    if hw > 1:
        for h in range(8):
            uh = q[0, h % tq, 16 * h:16 * h + 16].double()
            s = 0.25 * (K[:, :hw - 1, 16 * h:16 * h + 16].to(torch.bfloat16).double() @ uh)     # [blocks, hw - 1]
            lse = torch.logsumexp(s, dim=1)                                                    # sharpest logit: LSE
            K[:, hw - 1, 16 * h:16 * h + 16] = (4 * lse / uh.dot(uh)).view(-1, 1).float() * uh.float()
        V[:, hw - 1] += 12.0
    K, V = K.reshape(-1, 128).to(torch.bfloat16), V.reshape(-1, 128).to(torch.bfloat16)
    if shared:
        kv = torch.cat([K, V], dim=1)
        K, V = kv[:, :128], kv[:, 128:]
    blk = None if kv_block is None else torch.tensor(kv_block, dtype=torch.int32)
    return q, K, V, blk


def i2t_inputs(n: int, hw: int, tq: int, blocks: int, seed: int, q_block: list | None = None):
    """Q [blocks hw, 128], ktok, vtok [n, tq, 128] bf16, q_block int32 [n] or None.

    Adversarial: every valid logit is far below 0 (about -11 .. -40) while a padded token's would be 0 with value 0, so a
    padded token that leaked into the softmax would take all of it; head h's values are offset by 2h - 7, and block
    b's rows are 1 + b / 2 times as long, so its logits differ from another block's."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(8, 16, generator=g)
    u = u / u.norm(dim=1, keepdim=True)
    Q = u.reshape(1, 128) * (4 + torch.rand(blocks * hw, 128, generator=g)) + 0.1 * torch.randn(blocks * hw, 128, generator=g)
    Q = Q * (1 + 0.5 * torch.arange(blocks)).repeat_interleave(hw).view(-1, 1)
    depth = 12 + 6 * torch.rand(n, tq, 8, generator=g)                   # -(logit) per (token, head), at |Q_h| ~ 4.5
    ktok = -(depth / (0.25 * 4.5)).repeat_interleave(16, dim=2) * u.reshape(1, 1, 128)
    ktok = ktok + 0.05 * torch.randn(n, tq, 128, generator=g)
    vtok = torch.randn(n, tq, 128, generator=g) + _head_offsets()
    blk = None if q_block is None else torch.tensor(q_block, dtype=torch.int32)
    return Q.to(torch.bfloat16), ktok.to(torch.bfloat16), vtok.to(torch.bfloat16), blk


def ln_row_inputs(m: int, offset: float, res_rows: int, res_fp32: bool, seed: int, K: int = 128, N: int = 256):
    """a [m, K] bf16, w [N, K] bf16, bias, residual [res_rows, N] (fp32 or bf16, rows offset by `offset` plus a
    per-row level so block-mapped rows differ), gamma, beta."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(m, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.1
    res = torch.randn(res_rows, N, generator=g) * (1 + torch.rand(res_rows, 1, generator=g)) + offset
    res = res if res_fp32 else res.to(torch.bfloat16)
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g), 0.1 * torch.randn(N, generator=g)
    return a, w, bias, res, gamma, beta


def upscale_inputs(n: int, h: int, w: int, seed: int, cin: int = 256):
    """The upscaler's tensors in the decoder's layouts: keys bf16 [n h w, cin]; the ConvTranspose2d weights
    (w1 [cin, cin/4, 2, 2], w2 [cin/4, cin/8, 2, 2]) and biases; LN gamma / beta; hyper [n, cin/8]."""
    g = torch.Generator().manual_seed(seed)
    c4, c8 = cin // 4, cin // 8
    keys = torch.randn(n * h * w, cin, generator=g).to(torch.bfloat16)
    w1 = (torch.randn(cin, c4, 2, 2, generator=g) * cin ** -0.5).to(torch.bfloat16).float()
    b1 = 0.1 * torch.randn(c4, generator=g)
    gamma, beta = 1 + 0.2 * torch.randn(c4, generator=g), 0.3 * torch.randn(c4, generator=g)
    w2 = (torch.randn(c4, c8, 2, 2, generator=g) * c4 ** -0.5).to(torch.bfloat16).float()
    b2 = 0.3 * torch.randn(c8, generator=g)
    hyper = torch.randn(n, c8, generator=g)
    return dict(keys=keys, w1=w1, b1=b1, gamma=gamma, beta=beta, w2=w2, b2=b2, hyper=hyper)


def upscale2_inputs(P: int, h: int, w: int, seed: int, one_hot: bool = False):
    """up1 bf16 [P h w 4, 64], up2_w bf16 [128, 64] (GEMM layout), up2_b, hyper [P, 32].

    Adversarial for the GELU: the pre-activations sit near +-2.7, where erf and tanh GELU differ most (4.7e-4), and
    hyper is positive, so that difference adds up over the 32 channels.  one_hot: hyper[p] = e_(p mod 32), so every
    mask pixel is one GELU value of one (row, tap2) and a misplaced pixel shows."""
    g = torch.Generator().manual_seed(seed)
    up1 = (0.25 * torch.randn(P * h * w * 4, 64, generator=g)).to(torch.bfloat16)
    w2 = (torch.randn(64, 32, 2, 2, generator=g) * 64 ** -0.5).to(torch.bfloat16).float()
    sign = torch.where(torch.rand(32, generator=g) < 0.5, -1.0, 1.0)
    b2 = sign * (2.7 + 0.1 * torch.randn(32, generator=g))
    if one_hot:
        hyper = F.one_hot(torch.arange(P) % 32, 32).float()
    else:
        hyper = 0.2 + torch.rand(P, 32, generator=g)
    return up1, convt_gemm_weight(w2).to(torch.bfloat16), convt_gemm_bias(b2), hyper


def fused_inputs(n: int, hw: int, tq: int, seed: int):
    """Operands of t2i_fused and i2t_fused on coarse grids (keys and positional terms multiples of 1/4, weights of
    1/64, biases of 1/256), so every projection sum is exact in fp32 and the kernel's bf16 K | V and Q equal the
    reference's: the comparison then measures the attention and LayerNorm arithmetic alone."""
    g = torch.Generator().manual_seed(seed)
    grid = lambda t, s: (torch.round(t * s) / s)  # noqa: E731
    keys = grid(torch.randn(n * hw, 256, generator=g), 4).to(torch.bfloat16)
    kvw = grid(0.06 * torch.randn(256, 256, generator=g), 64).to(torch.bfloat16)
    kvb = grid(0.1 * torch.randn(256, generator=g), 256)
    pe_kv = torch.zeros(hw, 256)
    pe_kv[:, :128] = grid(torch.randn(hw, 128, generator=g), 4)          # the decoder's layout: the v half is 0
    q = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    wq = grid(0.06 * torch.randn(128, 256, generator=g), 64).to(torch.bfloat16)
    qb = grid(0.1 * torch.randn(128, generator=g), 256)
    pe_q = grid(torch.randn(hw, 128, generator=g), 4).to(torch.bfloat16)
    ktok = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    vtok = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    wo = (0.09 * torch.randn(256, 128, generator=g)).to(torch.bfloat16)
    ob = 0.1 * torch.randn(256, generator=g)
    ln = (1.0 + 0.1 * torch.randn(256, generator=g), 0.1 * torch.randn(256, generator=g), 1e-6)
    return dict(q=q, keys=keys, kvw=kvw, kvb=kvb, pe_kv=pe_kv.to(torch.bfloat16), wq=wq, qb=qb, pe_q=pe_q, ktok=ktok,
                vtok=vtok, wo=wo, ob=ob, ln=ln)


def t2i_fused_ref_tol(q, keys, kvw, kvb, pe_kv, hw: int):
    """(reference, tolerance) of t2i_fused: the t2i bound on the (exactly reproduced) bf16 K | V."""
    kv = rb(keys.to(D) @ kvw.to(D).t() + kvb.to(D) + pe_kv.to(D).repeat(keys.shape[0] // hw, 1))
    ref = t2i(q, kv[:, :128], kv[:, 128:], hw)
    return ref, t2i_tol(q, kv[:, :128], kv[:, 128:], hw, ref)


def i2t_fused_ref_tol(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln: tuple, hw: int):
    """(reference, tolerance) of i2t_fused.  The kernel's attention output differs from the reference's by the i2t
    bound plus both sides' bf16 rounding; that difference enters the out_proj (an fp32 sum of 128 products), whose
    sum with ob and the keys goes through the LayerNorm bound, then the bf16 output rounding."""
    g, b, eps = ln
    Q = rb(keys.to(D) @ wq.to(D).t() + qb.to(D) + pe_q.to(D).repeat(keys.shape[0] // hw, 1))
    att = i2t(Q, ktok, vtok, hw)
    datt = i2t_tol(Q, ktok, vtok, hw, att) + U8 * att.abs()
    att = rb(att)
    woa = wo.to(D).abs().t()
    x = att @ wo.to(D).t() + ob.to(D) + keys.to(D)
    ref = F.layer_norm(x, (256,), g.to(D), b.to(D), eps)
    dx = datt @ woa + 128 * U24 * (att.abs() @ woa) + 3 * U24 * x.abs().amax(-1, keepdim=True)
    return ref, _ln_err(x, dx, g, eps) + 3 * U24 * ref.abs() + U8 * ref.abs() + 1e-30


def swap_heads(x: torch.Tensor) -> torch.Tensor:
    """Heads h and h ^ 1 exchanged in the last dim (8 heads x 16)."""
    return x.reshape(*x.shape[:-1], 4, 2, 16).flip(-2).reshape(x.shape)


def max_ratio(err: torch.Tensor, tol: torch.Tensor) -> float:
    return (err.to(D) / tol.to(D)).max().item()
