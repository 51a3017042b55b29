"""Float64 restatements of the standard GEMM epilogue and of the encoder's LayerNorm (include/rsp_b200.h:
rsp_gemm_bf16 with epi_mode 0, rsp_conv3x3_nhwc_bf16, rsp_layernorm).  TEST INFRASTRUCTURE ONLY.

Rounding points of each kernel, in the order they happen:
  * gemm_bf16_wgmma_v2_kernel, standard epilogue (gemm_v2.cu, every schedule): bf16 A and W, exact products, an fp32
    accumulator over K taken by the tensor cores in k16 steps (aligned to the largest term and truncated, so c = 2 in
    c K U24 sum|a||w|); then, on the fp32 accumulator, one IEEE add of the fp32 bias, the activation (gelu_fast:
    within GELU_FAST_ERR of GELU(erf); ReLU: exact), one IEEE add of the fp32 or bf16 residual, and the output: fp32 as
    is, bf16 by round-to-nearest-even.  The implicit 3x3 convolution is the same GEMM over K = 9 C (zero halo).
  * layernorm_rows_kernel (rowops.cu): one warp per row; each lane sums its <= 4 MAXV values in order (MAXV = 2, 6,
    10 for C <= 256, 768, 1280), then 5 shuffle levels; mean = sum / C; the variance is a second pass over d = x - mean
    (two-pass, so a large common offset does not cancel), summed the same way; rstd = rsqrtf(var / C + eps) (2 ulp);
    y = (x - mean) rstd gamma + beta; GELU by gelu_erf (erff, 2 ulp); bf16 (RNE) or fp32 out.

``exact_operands`` builds A and W as small integers times powers of two, so that every product and every partial sum
is an integer multiple of 2^-F below 2^(23 - F) in magnitude: an fp32 sum of them is exact in any order, including
the tensor cores' truncating alignment.  On such operands the kernel's bytes are defined: ``gemm_expect`` gives them
(for GELU the interval the bytes must lie in).  ``gemm_std_tol`` and ``layernorm_rows_tol`` bound |kernel - reference|
element by element on real-valued operands, in the terms of oracle/decoder_kernels.py: U8 / U24 the unit roundoffs of
bf16 / fp32."""
from __future__ import annotations

import torch

from .decoder_kernels import D, GELU_FAST_ERR, GELU_LIP, U8, U24, gelu_erf64, max_ratio  # noqa: F401

F_BITS = 10          # exact operands: every value is an integer multiple of 2^-F_BITS
ROW_CHUNK = 8192     # rows per float64 block of the references


# ---------------------------------------------------------------------------------------------------- GEMM
def residual_rows(orow: torch.Tensor, res_mod: int = 0, res_block_map=None, res_block_rows: int = 0) -> torch.Tensor:
    """The residual row the epilogue reads for destination row orow (gemm.h)."""
    if res_block_map is not None:
        blk = torch.div(orow, res_block_rows, rounding_mode="floor")
        return res_block_map.to(orow.device).long()[blk] * res_block_rows + orow % res_block_rows
    return orow % res_mod if res_mod else orow


def _epilogue(acc, cols, bias, act, residual, rrow, fp32_steps: bool):
    x = acc if bias is None else acc + bias.to(D)
    if fp32_steps:
        x = x.float().to(D)
    if act == "gelu":
        x = gelu_erf64(x)
    elif act == "relu":
        x = x.clamp_min(0)
    if residual is not None:
        x = x + residual[rrow][:, cols].to(D)
        if fp32_steps:
            x = x.float().to(D)
    return x


def gemm_std(a, w, bias=None, act=None, residual=None, res_mod: int = 0, res_block_map=None, res_block_rows: int = 0,
             row_map=None, out_rows: int | None = None, fp32_steps: bool = False) -> torch.Tensor:
    """rsp_gemm_bf16 epi_mode 0: out[row_map[m], n] = act(sum_k a[m, k] w[n, k] + bias[n]) + residual[rrow, n] with
    rrow from the destination row (residual_rows).  float64 [out_rows, N], NaN where no row lands.  fp32_steps rounds
    to fp32 after the bias add and after the residual add, as the kernel does (exact operands: its bytes)."""
    M, N = a.shape[0], w.shape[0]
    out = torch.full((M if out_rows is None else out_rows, N), float("nan"), dtype=D, device=a.device)
    wd = w.to(D).t()
    cols = torch.arange(N, device=a.device)
    for m0 in range(0, M, ROW_CHUNK):
        rows = torch.arange(m0, min(M, m0 + ROW_CHUNK), device=a.device)
        dst = rows if row_map is None else row_map.to(a.device)[rows].long()
        keep = dst >= 0
        rows, dst = rows[keep], dst[keep]
        acc = a[rows].to(D) @ wd
        rrow = residual_rows(dst, res_mod, res_block_map, res_block_rows) if residual is not None else None
        assert rrow is None or len(rrow) == 0 or int(rrow.max()) < residual.shape[0], "residual row out of range"
        out[dst] = _epilogue(acc, cols, bias, act, residual, rrow, fp32_steps)
    return out


def gemm_expect(a, w, bias=None, act=None, residual=None, out_dtype=torch.bfloat16, **rmap):
    """(lo, hi) in out_dtype: the bytes the kernel must write on exact operands (lo == hi for act None / relu), or the
    interval they must lie in for GELU: gelu_fast within GELU_FAST_ERR + 4 U24 |GELU| of GELU(erf) of the exact
    pre-activation, then the residual add and the output rounding, both monotone.  NaN where no row lands."""
    if act != "gelu":
        e = gemm_std(a, w, bias, act, residual, fp32_steps=True, **rmap).float().to(out_dtype)
        return e, e
    assert rmap.get("res_block_map") is None, "GELU with a residual block map is not restated"
    pre = gemm_std(a, w, bias, None, None, fp32_steps=True, row_map=rmap.get("row_map"), out_rows=rmap.get("out_rows"))
    g = gelu_erf64(pre)
    t = GELU_FAST_ERR + 4 * U24 * g.abs()
    lo, hi = g - t, g + t
    if residual is not None:
        orow = torch.arange(pre.shape[0], device=pre.device)
        r = residual[residual_rows(orow, rmap.get("res_mod", 0), rmap.get("res_block_map"),
                                   rmap.get("res_block_rows", 0)).clamp(0, residual.shape[0] - 1)][:, :pre.shape[1]]
        lo, hi = lo + r.to(D), hi + r.to(D)
        lo, hi = lo - 2 * U24 * lo.abs(), hi + 2 * U24 * hi.abs()
    return lo.float().to(out_dtype), hi.float().to(out_dtype)


def gemm_std_tol(a, w, bias=None, act=None, residual=None, ref=None, out_bf16: bool = True, **rmap) -> torch.Tensor:
    """Bound on |kernel - gemm_std| for real-valued operands: 2 K U24 sum|a||w| (the tensor cores' truncating fp32
    accumulation), U24 |acc + bias| for the bias add, the activation (GELU: Lipschitz GELU_LIP, GELU_FAST_ERR and its
    own rounding; ReLU: Lipschitz 1), U24 |out| for the residual add, and the output rounding (U8 or U24 |ref|)."""
    K = a.shape[1]
    sel = dict(row_map=rmap.get("row_map"), out_rows=rmap.get("out_rows"))
    mag = gemm_std(a.abs(), w.abs(), **sel)
    pre = gemm_std(a, w, bias, None, None, **sel)
    e = 2 * K * U24 * mag + U24 * pre.abs()
    if act == "gelu":
        e = GELU_LIP * e + GELU_FAST_ERR + 2 * U24 * gelu_erf64(pre).abs()
    if residual is not None:
        e = e + U24 * ref.abs()
    return e + (U8 if out_bf16 else U24) * ref.abs() + 1e-30


def _grid(shape, lim: int, g: torch.Generator, scale_bits: int) -> torch.Tensor:
    """Integers in [-lim, lim] times 2^-scale_bits (times 1, 1/2 or 1/4 per element)."""
    i = torch.randint(-lim, lim + 1, shape, generator=g, device=g.device).float()
    e = torch.randint(0, 3, shape, generator=g, device=g.device).float()
    return i * torch.exp2(-e - scale_bits)


def exact_operands(M: int, N: int, K: int, seed: int, *, bias: bool = True, residual: str | None = None,
                   res_rows: int | None = None, res_cols: int | None = None, lda: int | None = None,
                   ldw: int | None = None, pad_value: float = float("nan"), device="cuda"):
    """a bf16 [M, K] (row stride lda), w bf16 [N, K] (row stride ldw), bias fp32 [N] or None, residual or None.

    a = i 2^-e (|i| <= 7, e in 0..2), w = i 2^-(e + 6): every product is a multiple of 2^-F_BITS of at most 784
    units, so a sum of K <= 4096 of them stays below 2^22 units, bias and residual included (fp32 keeps 24 bits):
    exact in any order and under truncating alignment, with bits to spare.  bias is a multiple of 2^-F_BITS below 4 in
    magnitude.  residual: "grid" fp32 on the same grid, "bf16" bf16 multiples of 2^-8 below 1 (exact after any
    add), "fp32" arbitrary fp32 (its add is the one rounding).  The padding columns of lda / ldw hold pad_value."""
    g = torch.Generator(device=device).manual_seed(seed)
    ri = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g, device=device)  # noqa: E731
    lda, ldw = lda or K, ldw or K
    A = torch.full((M, lda), pad_value, dtype=torch.bfloat16, device=device)
    A[:, :K] = _grid((M, K), 7, g, 0).to(torch.bfloat16)
    Wt = torch.full((N, ldw), pad_value, dtype=torch.bfloat16, device=device)
    Wt[:, :K] = _grid((N, K), 7, g, 6).to(torch.bfloat16)
    b = (ri(-4096, 4097, (N,)).float() * 2.0 ** -F_BITS) if bias else None
    r = None
    if residual is not None:
        shape = (res_rows or M, res_cols or N)
        if residual == "grid":
            r = ri(-4096, 4097, shape).float() * 2.0 ** -F_BITS
        elif residual == "bf16":
            r = (ri(-255, 256, shape).float() * 2.0 ** -8).to(torch.bfloat16)
        else:
            r = torch.randn(shape, generator=g, device=device) * torch.exp2(ri(-12, 4, shape).float())
    return A[:, :K], Wt[:, :K], b, r


# ---------------------------------------------------------------------------------------------------- LayerNorm
def lanes_per_value(C: int) -> int:
    """Values one lane of layernorm_rows_kernel sums before the shuffles: 4 per 128-column step of its MAXV."""
    return 4 * ((C + 127) // 128)


def _ln_src(x, src_map):
    xd = x.to(D)
    if src_map is None:
        return xd, None
    s = src_map.to(x.device).long()
    return xd[s.clamp_min(0)], s < 0


def layernorm_rows(x, gamma, beta, eps: float, src_map=None, gelu: bool = False) -> torch.Tensor:
    """rsp_layernorm: out[i] = LN(x[src_map[i]]) gamma + beta (then GELU(erf)), zeros where src_map[i] < 0; float64."""
    xs, pad = _ln_src(x, src_map)
    mu = xs.mean(-1, keepdim=True)
    var = ((xs - mu) ** 2).mean(-1, keepdim=True)
    y = (xs - mu) / torch.sqrt(var + eps) * gamma.to(D) + beta.to(D)
    if gelu:
        y = gelu_erf64(y)
    if pad is not None:
        y[pad] = 0
    return y


def layernorm_rows_tol(x, gamma, beta, eps: float, ref, out_bf16: bool, src_map=None, gelu: bool = False):
    """Bound on |kernel - layernorm_rows| from layernorm_rows_kernel's rounding points (L = lanes_per_value(C)):
      * the fp32 sum over L values then 5 shuffle levels, and the division: dmu <= (L + 6) U24 mean|x|;
      * the two-pass variance over d = x - mean_hat: sum (x - mean_hat)^2 = C var + C dmu^2 exactly, and the
        rounded d, d^2, L + 5 sums and the division add (L + 9) U24 of it;
      * var / C + eps, rsqrtf (2 ulp): rstd carries dvar / (2 (var + eps)) + 6 U24 relative;
      * y = (x - mean) rstd g + b: |g| rstd (dmu + |x - mu| drstd) + 4 U24 (|g xhat| + |b|);
      * GELU: GELU_LIP dy + 8 U24 |y| (erff 2 ulp, 1 + erf, 0.5 x products);
      * the output: U8 |ref| (bf16) or U24 |ref| (fp32)."""
    xs, pad = _ln_src(x, src_map)
    C = xs.shape[-1]
    L = lanes_per_value(C)
    mu = xs.mean(-1, keepdim=True)
    var = ((xs - mu) ** 2).mean(-1, keepdim=True)
    r = (var + eps).rsqrt()
    dmu = (L + 6) * U24 * xs.abs().mean(-1, keepdim=True)
    dvar = (L + 9) * U24 * (var + dmu ** 2) + dmu ** 2
    dr = dvar / (2 * (var + eps)) + 6 * U24
    g, b = gamma.to(D).abs(), beta.to(D).abs()
    xhat = (xs - mu).abs() * r
    y = xhat * g + b
    e = g * r * (dmu + (xs - mu).abs() * dr) + 4 * U24 * y
    if gelu:
        e = GELU_LIP * e + 8 * U24 * y
    e = e + (U8 if out_bf16 else U24) * ref.abs() + 1e-30
    if pad is not None:
        e[pad] = 1e-30
    return e
