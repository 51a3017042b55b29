"""Float64 restatements of the ViT encoder's attention kernels (include/rsp_b200.h: rsp_vit_attention with and
without out_row_map, rsp_vit_attention_simt and the three-pass path of rsp_split_heads, rsp_transpose_cols,
rsp_attn_softmax_bias and two grouped GEMMs).  TEST INFRASTRUCTURE ONLY.

``attention`` is SamVisionAttention's core (HF:803-831, rel-pos HF:729-801) in float64 on the kernels' layout: qkv
[n_seq*T, 3*H*hd] with columns [q | k | v], heads contiguous inside each; out [n_seq*T, H*hd].  The scale hd^-0.5
multiplies q.k only; the decomposed rel-pos bias uses the unscaled q.  The softmax is float64 too (restate's
vit_attention_core runs it in fp32), and the output is returned unrounded: a tolerance includes the kernel's own bf16
output rounding.  Work is chunked over (sequence, head) pairs so that ViT-H global attention (16 heads, T = 4096)
fits, and runs on the device of its inputs.

``flash_tol``, ``simt_tol`` and ``three_pass_tol`` bound |kernel - reference| element by element from each path's
rounding points.  Per query row, with exact softmax weights w_j and per-key logit errors ds_j (natural log units):
  * q.k and q.table are fp32 sums of hd products: ds_j <= c hd U24 A_j, A_j = hd^-0.5 |q|.|k_j| + |q|.|Rh| + |q|.|Rw|
    (c = 2 on the tensor cores, whose fp32 accumulation truncates, 1 on CUDA cores); the log2 e multiplies, the fma
    and the subtraction of the row max add a few U24 of |logit| and |logit - max|;
  * each weight goes through one exp (ex2.approx.ftz or expf, within EX2_REL) and, on the online-softmax paths, a
    rounded rescale per key tile (flash) or key (SIMT) - the same factor multiplies the output and the row sum;
  * a logit error moves a softmax-weighted mean by at most 2 (sum_j w_j ds_j) max|V|;
  * flash: P is rounded to fp16 (U11 relative, 2^-25 absolute below 2^-14) while the row sum l is over the unrounded
    P; V is converted bf16 -> fp16, exact for 2^-14 <= |v| <= 65280, 2^-25 absolute below; P V is an fp32 sum of T;
  * three-pass: P = bf16(p / l) is normalised before rounding, so the rounded row does not sum to 1 (U8 of sum P|v|);
    P V is a bf16 x bf16 GEMM with fp32 accumulation over T keys;
  * every path rounds its output to bf16 (U8 |out|).
The builders make the adversarial inputs the CPU and GPU tests share."""
from __future__ import annotations

import zlib

import torch

from oracle.decoder_kernels import U8, U24, max_ratio  # noqa: F401  (max_ratio: re-exported for the tests)

D = torch.float64
U11 = 2.0 ** -11            # fp16 unit roundoff (11 significant bits)
EX2_REL = 2.0 ** -21        # relative error of ex2.approx.ftz.f32 and expf (PTX / CUDA: 2 ulp), with margin
FP16_V_MAX = 65280.0        # largest bf16 value that converts to a finite fp16
PAIR_BUDGET = 1 << 25       # float64 logits per chunk: 256 MB
BN = 64                     # keys per tile of the flash kernel


def rel_index(S: int, device=None) -> torch.Tensor:
    """idx[a, b] = a - b + S - 1: the table row of query coordinate a and key coordinate b (HF:729-758)."""
    a = torch.arange(S, device=device)
    return a[:, None] - a[None, :] + S - 1


def _logits(q: torch.Tensor, k: torch.Tensor, Rh: torch.Tensor, Rw: torch.Tensor, S: int, scale: float) -> torch.Tensor:
    """scale q k^T + q.Rh[qh - kh + S - 1] + q.Rw[qw - kw + S - 1]: q, k [n, T, hd]; Rh, Rw gathered [S, S, hd]."""
    n, T, hd = q.shape
    q4 = q.reshape(n, S, S, hd)
    bh = torch.einsum("nhwc,hkc->nhwk", q4, Rh)          # [n, qh, qw, kh]
    bw = torch.einsum("nhwc,wkc->nhwk", q4, Rw)          # [n, qh, qw, kw]
    s = (q * scale) @ k.transpose(1, 2)
    return (s.view(n, S, S, S, S) + bh[..., :, None] + bw[..., None, :]).view(n, T, T)


def blocks(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int, with_abs: bool = False):
    """Yields (seq, head, v, logits, A) per chunk of (sequence, head) pairs: seq / head int64 [n]; v float64 [n, T, hd];
    logits float64 [n, T, T] (natural log units); A = the same sums over |operands| (the scale of the logits' rounding
    error) when with_abs, else None."""
    T = S * S
    x = qkv.reshape(n_seq, T, 3, H, hd)
    idx = rel_index(S, qkv.device)
    Rh, Rw = rel_h.to(D)[idx], rel_w.to(D)[idx]
    scale = hd ** -0.5
    per = max(1, PAIR_BUDGET // (T * T))
    for b0 in range(0, n_seq * H, per):
        b = torch.arange(b0, min(n_seq * H, b0 + per), device=qkv.device)
        seq, head = b // H, b % H
        q, k, v = (x[seq, :, i, head].to(D) for i in range(3))
        lg = _logits(q, k, Rh, Rw, S, scale)
        A = _logits(q.abs(), k.abs(), Rh.abs(), Rw.abs(), S, scale) if with_abs else None
        yield seq, head, v, lg, A


def _put(out: torch.Tensor, n_seq: int, T: int, H: int, hd: int, seq, head, val) -> None:
    out.view(n_seq, T, H, hd)[seq, :, head] = val


def attention(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int) -> torch.Tensor:
    """rsp_vit_attention in float64: [n_seq*T, 3*H*hd] -> [n_seq*T, H*hd], unrounded."""
    T = S * S
    out = torch.empty(n_seq * T, H * hd, dtype=D, device=qkv.device)
    for seq, head, v, lg, _ in blocks(qkv, rel_h, rel_w, n_seq, S, H, hd):
        _put(out, n_seq, T, H, hd, seq, head, torch.softmax(lg, dim=-1) @ v)
    return out


# ---------------------------------------------------------------------------------------------------- tolerances
def _tol(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int, ref: torch.Tensor, path: str) -> torch.Tensor:
    T = S * S
    nkt = (T + BN - 1) // BN
    dot = (2 * hd + 16) if path in ("flash", "three_pass") else (hd + 8)      # tensor-core sums truncate
    tol = torch.empty(n_seq * T, H * hd, dtype=D, device=qkv.device)
    for seq, head, v, lg, A in blocks(qkv, rel_h, rel_w, n_seq, S, H, hd, with_abs=True):
        smax = lg.amax(-1, keepdim=True)
        e = torch.exp(lg - smax)
        lsum = e.sum(-1, keepdim=True)                  # >= 1: the row sum relative to the row max
        w = e / lsum
        ds = dot * U24 * A + 3 * U24 * lg.abs() + 2 * U24 * (smax - lg)
        dsw = (w * ds).sum(-1, keepdim=True)
        vmax = v.abs().amax(dim=(1, 2)).view(-1, 1, 1)
        wabs = w @ v.abs()                              # sum_j w_j |v_j|: the scale of the P V rounding
        if path == "flash":   # per-tile rescales (2 roundings each, the same alpha on O and l), fp16 P and V
            dsw = dsw + EX2_REL + 2 * nkt * U24
            head_err = (2 * dsw * vmax + U11 * wabs + 2.0 ** -25 * T * vmax / lsum + 2.0 ** -24
                        + (2 * T + 2 * nkt + 8) * U24 * wabs)
            rel = U8 + (2 * T + 2 * nkt + 8) * U24
        elif path == "simt":  # one rescale per key (2 roundings), sequential fp32 sums
            dsw = dsw + EX2_REL + 2 * T * U24
            head_err = 2 * dsw * vmax + (2 * T + 4) * U24 * wabs
            rel = U8 + (2 * T + 4) * U24
        elif path == "three_pass":   # one exp, P normalised then rounded to bf16, P V over T on the tensor cores
            dsw = dsw + EX2_REL
            head_err = 2 * dsw * vmax + U8 * wabs + (3 * T + 8) * U24 * wabs
            rel = U8
        else:
            raise ValueError(path)
        refb = ref.view(n_seq, T, H, hd)[seq, :, head].abs()
        _put(tol, n_seq, T, H, hd, seq, head, head_err * (1 + U8) + rel * refb + 1e-30)
    return tol


def flash_tol(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int, ref: torch.Tensor) -> torch.Tensor:
    """Bound on |rsp_vit_attention - attention| for S = 14 / 32 / 64 (attention.cu, the wgmma kernel)."""
    return _tol(qkv, rel_h, rel_w, n_seq, S, H, hd, ref, "flash")


def simt_tol(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int, ref: torch.Tensor) -> torch.Tensor:
    """Bound on |rsp_vit_attention_simt - attention|: fp32 throughout, bf16 output."""
    return _tol(qkv, rel_h, rel_w, n_seq, S, H, hd, ref, "simt")


def three_pass_tol(qkv, rel_h, rel_w, n_seq: int, S: int, H: int, hd: int, ref: torch.Tensor) -> torch.Tensor:
    """Bound on |vit_attention - attention| on the three-pass path (S = 48 / 80, attention_generic.cu)."""
    return _tol(qkv, rel_h, rel_w, n_seq, S, H, hd, ref, "three_pass")


def softmax_bias(scores, tab, NT: int, S: int, scale: float, row0: int = 0) -> torch.Tensor:
    """rsp_attn_softmax_bias in float64 on rows row0 .. row0 + len(scores) of its input: scores fp32 [rows, >= T],
    tab fp32 [rows, >= 2 NT] -> P [rows, T] = softmax_k(scale scores[r, k] + tab[r, qh - kh + S - 1]
    + tab[r, NT + qw - kw + S - 1]), query q = r % T."""
    return torch.softmax(_softmax_bias_logits(scores, tab, NT, S, scale, row0)[0], dim=-1)


def _softmax_bias_logits(scores, tab, NT: int, S: int, scale: float, row0: int):
    T = S * S
    rows = scores.shape[0]
    q = (row0 + torch.arange(rows, device=scores.device)) % T
    qh, qw = q // S, q % S
    kk = torch.arange(S, device=scores.device)
    th = tab.to(D).gather(1, qh[:, None] - kk[None, :] + S - 1)             # [rows, kh]
    tw = tab.to(D).gather(1, NT + qw[:, None] - kk[None, :] + S - 1)        # [rows, kw]
    sc = scores[:, :T].to(D) * scale
    bias = (th[:, :, None] + tw[:, None, :]).reshape(rows, T)
    return sc + bias, sc, bias


def softmax_bias_tol(scores, tab, NT: int, S: int, scale: float, ref: torch.Tensor, row0: int = 0) -> torch.Tensor:
    """Bound on |rsp_attn_softmax_bias - softmax_bias|: the logit in base 2 by one fma of fp32 terms (scale and the
    log2 e products rounded), ex2.approx, an fp32 row sum of T terms, P = bf16(p / l)."""
    T = S * S
    lg, sc, bias = _softmax_bias_logits(scores, tab, NT, S, scale, row0)
    smax = lg.amax(-1, keepdim=True)
    ds = 4 * U24 * (sc.abs() + bias.abs() + lg.abs()) + 2 * U24 * (smax - lg)
    w = ref
    dsw = (w * ds).sum(-1, keepdim=True)
    rel = ds + dsw + EX2_REL + (T + 6) * U24
    return w * rel * (1 + U8) + U8 * w * (1 + rel) + 2.0 ** -125      # ex2.approx.ftz flushes p < 2^-126 to 0


def softmax_bias_inputs(S: int, n_rows: int, NT: int, lds: int, ldt: int, seed: int):
    """fp32 scores [n_rows, lds] ~ 6 N(0, 1) and tab [n_rows, ldt] ~ 2 N(0, 1) in the columns the kernel reads; NaN
    in every other column (past T, between 2S - 1 and NT, past 2 NT), so a stray read shows."""
    T = S * S
    g = torch.Generator().manual_seed(seed)
    scores = torch.full((n_rows, lds), float("nan"))
    scores[:, :T] = 6.0 * torch.randn(n_rows, T, generator=g)
    tab = torch.full((n_rows, ldt), float("nan"))
    tab[:, :2 * S - 1] = 2.0 * torch.randn(n_rows, 2 * S - 1, generator=g)
    tab[:, NT:NT + 2 * S - 1] = 2.0 * torch.randn(n_rows, 2 * S - 1, generator=g)
    return scores, tab


# ---------------------------------------------------------------------------------------------------- input builders
KINDS = ("random", "tables15", "sharp", "last_key", "rising", "one_hot", "uniform", "offset", "p_tie", "fp16_edge")
ONE_HOT_LOGIT = 40.0        # table entry of the one-hot inputs: every other key is >= 40 below the attended one


def seed_of(*key) -> int:
    return zlib.crc32(repr(key).encode())


def inputs(kind: str, n_seq: int, S: int, H: int, hd: int, seed: int | None = None):
    """qkv bf16 [n_seq*T, 3*H*hd], rel_h, rel_w bf16 [2S-1, hd] on the CPU, one adversarial case per kind:
      random     q, k, v ~ N(0, 1), tables at 0.2;
      tables15   the same with tables at 1.5 (the rel-pos terms dominate the logits);
      sharp      q and k of each (sequence, head) scaled by 3..8: near one-hot rows, large fp32 logits;
      last_key   the sharpest logit of every (query, head) in the last valid key T-1 (key 195 of a window, the last key
                 tile of S = 32 / 64), whose value is offset by +12;
      rising     the logits rise by ~1.5 per 64-key tile, so the running max moves in every tile; V offset by +2;
      one_hot    one-hot tables: query (qh, qw) attends only to key (qh, qw), every other logit is >= 40 lower, so the
                 output row is that key's v exactly (|v| >= 0.05, inside fp16's normal range);
      uniform    q = 0 and zero tables: a uniform softmax, the output is the mean of V;
      offset     V = c_h + 0.05 N(0, 1) with |c_h| up to 16 H: the output cancels against large values;
      p_tie      every row the same: key 0 at logit 0 with v = 0, the others at P = 1/2 + 2^-9 -+ 2^-13 (just below /
                 above a bf16 rounding tie) with v = +1 / -1, so bf16 rounding of P would push every term the same way
                 while the output cancels to about 0;
      fp16_edge  head 0 has |v| = 65280 (the largest bf16 that stays finite in fp16) in some keys, head H-1 (H > 1)
                 has |v| ~ 1e-6, inside fp16's subnormal range."""
    if kind not in KINDS:
        raise ValueError(kind)
    g = torch.Generator().manual_seed(seed_of(kind, n_seq, S, H, hd) if seed is None else seed)
    T = S * S
    q = torch.randn(n_seq, T, H, hd, generator=g)
    k = torch.randn(n_seq, T, H, hd, generator=g)
    v = torch.randn(n_seq, T, H, hd, generator=g)
    tab = 1.5 if kind == "tables15" else 0.2
    rh = tab * torch.randn(2 * S - 1, hd, generator=g)
    rw = tab * torch.randn(2 * S - 1, hd, generator=g)
    scale = hd ** -0.5
    if kind == "sharp":
        f = 3.0 + 5.0 * torch.rand(n_seq, 1, H, 1, generator=g)
        q, k = q * f, k * f
    elif kind == "last_key":
        rh, rw = rh * 0.25, rw * 0.25
        u = torch.randn(n_seq, 1, H, hd, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        q = 3.0 * u + 0.3 * q
        qn = q.to(torch.bfloat16).double()
        qu = (qn * u.double()).sum(-1).amin(1)                                  # [n_seq, H], > 0
        # every other logit <= |q| (scale max|k| + max|Rh| + max|Rw|); the last key's >= scale beta q.u - |q| (..)
        kmax = k.to(torch.bfloat16).double().norm(dim=-1).amax(1)
        rmax = rh.to(torch.bfloat16).double().norm(dim=-1).amax() + rw.to(torch.bfloat16).double().norm(dim=-1).amax()
        qmax = qn.norm(dim=-1).amax(1)
        other = qmax * (scale * kmax + rmax)
        beta = (other + qmax * rmax + 1.0) / (scale * qu)
        k[:, T - 1] = (beta.unsqueeze(-1) * u[:, 0]).float()
        v[:, T - 1] += 12.0
    elif kind == "rising":
        rh, rw = rh * 0.25, rw * 0.25
        u = torch.randn(n_seq, 1, H, hd, generator=g)
        u = u / u.norm(dim=-1, keepdim=True)
        q = 4.0 * u + 0.1 * q
        slope = 1.5 / (BN * scale * 4.0)                                       # ~1.5 per 64-key tile
        j = torch.arange(T, dtype=torch.float32).view(1, T, 1, 1)
        k = slope * j * u + 0.1 * k
        v = v + 2.0
    elif kind == "one_hot":
        q = torch.zeros_like(q)
        q[..., 0] = 1.0
        q[..., 1] = 1.0
        k[..., :2] = 0.0
        rh, rw = torch.zeros(2 * S - 1, hd), torch.zeros(2 * S - 1, hd)
        rh[S - 1, 0] = ONE_HOT_LOGIT
        rw[S - 1, 1] = ONE_HOT_LOGIT
        v = torch.sign(v) * (0.05 + v.abs())
        v[v == 0] = 0.05
    elif kind == "uniform":
        q = torch.zeros_like(q)
        rh, rw = torch.zeros(2 * S - 1, hd), torch.zeros(2 * S - 1, hd)
    elif kind == "offset":
        c = torch.tensor([(-1.0) ** h * 16.0 * (h + 1) for h in range(H)]).view(1, 1, H, 1)
        v = c + 0.05 * v
    elif kind == "p_tie":
        q = torch.zeros_like(q)
        q[..., :2] = 1.0
        rh, rw = torch.zeros(2 * S - 1, hd), torch.zeros(2 * S - 1, hd)
        j = torch.arange(T)
        pos = j % 2 == 1
        p = torch.where(pos, 0.5 + 2.0 ** -9 - 2.0 ** -13, 0.5 + 2.0 ** -9 + 2.0 ** -13).double()
        p[0] = 1.0
        s = torch.log(p) / scale                      # q.k = k0 + k1, two bf16 terms: within 2^-16 of s
        k0 = s.to(torch.bfloat16).double()
        k1 = (s - k0).to(torch.bfloat16).double()
        k = torch.zeros_like(k)
        k[..., 0] = k0.float().view(1, T, 1)
        k[..., 1] = k1.float().view(1, T, 1)
        v = torch.where(pos, 1.0, -1.0).view(1, T, 1, 1).expand(n_seq, T, H, hd).clone()
        v[:, 0] = 0.0
    elif kind == "fp16_edge":
        hot = torch.rand(n_seq, T, hd, generator=g) < 0.02
        v[:, :, 0] = torch.where(hot, torch.sign(v[:, :, 0]) * FP16_V_MAX, v[:, :, 0])
        v[:, :, 0, 0] = FP16_V_MAX                                              # max|v| = 65280 in every sequence
        if H > 1:
            v[:, :, H - 1] = v[:, :, H - 1] * 1e-6
    qkv = torch.cat([q.reshape(n_seq * T, H * hd), k.reshape(n_seq * T, H * hd), v.reshape(n_seq * T, H * hd)], dim=1)
    return qkv.to(torch.bfloat16), rh.to(torch.bfloat16), rw.to(torch.bfloat16)


def window_inputs(batch: int, grid: int, H: int, hd: int, kind: str = "random", window: int = 14):
    """The windowed qkv the encoder feeds the kernel: rows of window padding tokens equal the qkv bias vector (LN1
    writes zero rows for them and the qkv GEMM adds its bias).  -> qkv bf16 [batch*nW*window^2, 3*H*hd], rel_h, rel_w,
    the window map of sam_encoder.window_maps (int32, -1 = padding) and n_win."""
    from rsprompter_b200.sam_encoder import window_maps
    wmap, n_win = window_maps(batch, grid, window, torch.device("cpu"))
    qkv, rh, rw = inputs(kind, batch * n_win, window, H, hd, seed=seed_of("window", kind, batch, grid, H, hd))
    g = torch.Generator().manual_seed(seed_of("bias", batch, grid, H, hd))
    bias = (0.5 * torch.randn(3 * H * hd, generator=g)).to(torch.bfloat16)
    qkv[wmap < 0] = bias
    return qkv, rh, rw, wmap, n_win
