"""The float64 references of the standard GEMM epilogue and the row LayerNorm (oracle/gemm_kernels.py), checked
without a GPU:
  * the exact operands are exact: fp32 sums in sequential, pairwise and 16-wide blocked order, and a tensor-core-like
    sum that aligns each k16 group to its largest term and truncates to a 24-bit window, all equal the float64 sum;
  * each bound holds for an fp32 emulation of the kernel's rounding points, and each named defect, restated on the
    emulation, falls outside it;
  * the row kernels' entry points reject arguments their accesses cannot take, before anything is launched."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_kernels as gk

D = torch.float64


def _seq_sum(a, w):
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
    for k in range(a.shape[1]):
        acc = acc + a[:, k:k + 1].float() * w[:, k].float()
    return acc


def _blocked_sum(a, w, block=16):
    K = a.shape[1]
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
    for k0 in range(0, K, block):
        part = (a[:, None, k0:k0 + block].float() * w[None, :, k0:k0 + block].float()).sum(-1)
        acc = acc + part
    return acc


def _truncating_sum(a, w, window=24, group=16):
    """Per k16 group: the products and the running sum aligned to the largest of them, each truncated toward zero to
    multiples of 2^(e_max - window + 1), summed exactly, then rounded to fp32."""
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=D)
    for k0 in range(0, a.shape[1], group):
        terms = a[:, None, k0:k0 + group].to(D) * w[None, :, k0:k0 + group].to(D)
        terms = torch.cat([terms, acc[..., None]], dim=-1)
        emax = torch.frexp(terms.abs().amax(-1, keepdim=True).clamp_min(1e-300)).exponent.to(D)
        q = torch.exp2(emax - window)
        acc = (torch.trunc(terms / q) * q).sum(-1).float().to(D)
    return acc


@pytest.mark.parametrize("M,N,K", [(6, 5, 1288), (4, 3, 2304), (9, 7, 8)])
def test_exact_operands_sum_exactly_in_any_order(M, N, K):
    a, w, b, r = gk.exact_operands(M, N, K, seed=K, residual="grid", device="cpu")
    ref = a.to(D) @ w.to(D).t()
    assert torch.equal(ref, ref.float().to(D))                          # representable in fp32
    assert torch.equal(ref + b.to(D) + r.to(D), (ref + b.to(D) + r.to(D)).float().to(D))
    for got in (_seq_sum(a, w), a.float() @ w.float().t(), _blocked_sum(a, w), _truncating_sum(a, w)):
        assert torch.equal(got.to(D), ref)
    # the truncating emulation is not vacuous: on real-valued operands it differs from the float64 sum
    g = torch.Generator().manual_seed(K)
    ar = torch.randn(M, K, generator=g).to(torch.bfloat16)
    wr = torch.randn(N, K, generator=g).to(torch.bfloat16)
    if K >= 64:
        assert not torch.equal(_truncating_sum(ar, wr, window=12), ar.to(D) @ wr.to(D).t())


def test_exact_operands_round_in_bf16():
    """The exact sums carry more than 8 significant bits, so the bf16 output rounding is exercised (ties included)."""
    a, w, b, _ = gk.exact_operands(512, 64, 256, seed=5, device="cpu")
    x = (a.to(D) @ w.to(D).t() + b.to(D)).float()
    rn = x.to(torch.bfloat16).float()
    tr = (x.view(torch.int32) & ~0xFFFF).view(torch.float32)
    assert (rn != x).float().mean() > 0.5 and (rn != tr).float().mean() > 0.3
    ties = ((x.view(torch.int32) & 0xFFFF) == 0x8000).sum().item()
    assert ties > 10


# ---------------------------------------------------------------------------------------------------- GEMM bound
def _real_operands(M, N, K, seed, res_rows):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16)
    b = torch.randn(N, generator=g)
    r = torch.randn(res_rows, N, generator=g)
    return a, w, b, r


def _emulate(a, w, b, act, r, rrow, out_bf16, *, trunc=False, acc_bf16=False, bias_after=False, res_before=False,
             k_used=None):
    """The standard epilogue in fp32 on CPU, with a defect switched on by each flag."""
    K = a.shape[1] if k_used is None else k_used
    x = a[:, :K].float() @ w[:, :K].float().t()
    if acc_bf16:
        x = x.to(torch.bfloat16).float()
    if not bias_after:
        x = x + b
    if res_before:
        x = x + r[rrow]
    if act == "gelu":
        x = F.gelu(x)
    elif act == "relu":
        x = torch.relu(x)
    if bias_after:
        x = x + b
    if not res_before:
        x = x + r[rrow]
    if not out_bf16:
        return x.to(D)
    if trunc:
        return (x.view(torch.int32) & ~0xFFFF).view(torch.float32).to(D)
    return x.to(torch.bfloat16).to(D)


@pytest.mark.parametrize("act", [None, "relu", "gelu"])
@pytest.mark.parametrize("out_bf16", [True, False])
def test_gemm_bound_holds_and_defects_fall_outside(act, out_bf16):
    M, N, K, res_mod = 256, 96, 200, 64
    a, w, b, r = _real_operands(M, N, K, seed=7, res_rows=M)     # rows >= res_mod are only read if it is ignored
    rows = torch.arange(M)
    rrow = rows % res_mod
    ref = gk.gemm_std(a, w, b, act, r, res_mod=res_mod)
    tol = gk.gemm_std_tol(a, w, b, act, r, ref, out_bf16, res_mod=res_mod)
    em = lambda **kw: _emulate(a, w, b, act, r, rrow, out_bf16, **kw)  # noqa: E731
    ratio = lambda got: gk.max_ratio((got - ref).abs(), tol)  # noqa: E731
    assert ratio(em()) <= 1.0
    defects = {
        "res_mod ignored": _emulate(a, w, b, act, r, rows, out_bf16),
        "residual row off by one": _emulate(a, w, b, act, r, (rrow + 1) % res_mod, out_bf16),
        "last k-block dropped": em(k_used=K // 64 * 64),
    }
    if act == "relu":
        defects["bias after the activation"] = em(bias_after=True)
        defects["residual before the activation"] = em(res_before=True)
    if out_bf16:
        defects["bf16 truncation"] = em(trunc=True)
    else:
        defects["accumulator rounded to bf16 before the bias"] = em(acc_bf16=True)
    for name, got in defects.items():
        assert ratio(got) > 1.0, name


# ---------------------------------------------------------------------------------------------------- LayerNorm
def _ln_emulate(x, gamma, beta, eps, out_bf16, gelu=False, *, one_pass=False, eps_outside=False, tanh=False,
                src_shift=0):
    """layernorm_rows_kernel in fp32: per-lane sequential sums over the lane's 4-value groups, 5 xor-shuffle levels,
    two-pass variance (or a defect switched on by each flag)."""
    rows, C = x.shape
    maxv = 2 if C <= 256 else 6 if C <= 768 else 10
    src = (torch.arange(rows) + src_shift) % rows
    v = torch.zeros(rows, maxv * 128, dtype=torch.float32)
    v[:, :C] = x[src].float()
    v = v.view(rows, maxv, 32, 4)

    def lane_sum(t):
        s = torch.zeros(rows, 32, dtype=torch.float32)
        for i in range(maxv):
            s = s + (((t[:, i, :, 0] + t[:, i, :, 1]) + t[:, i, :, 2]) + t[:, i, :, 3])
        for sh in (16, 8, 4, 2, 1):
            s = s + s[:, torch.arange(32) ^ sh]
        return s[:, :1]

    live = torch.zeros(maxv * 128, dtype=torch.bool)
    live[:C] = True
    live = live.view(maxv, 32, 4)
    mean = lane_sum(v) / C
    if one_pass:
        var = lane_sum(v * v) / C - mean * mean
    else:
        d = torch.where(live, v - mean[..., None, None], torch.zeros(()))
        var = lane_sum(d * d) / C
    rstd = 1.0 / (torch.sqrt(var) + eps) if eps_outside else torch.rsqrt(var + eps)
    y = ((v.view(rows, -1)[:, :C] - mean) * rstd) * gamma + beta
    if gelu:
        y = F.gelu(y, approximate="tanh" if tanh else "none")
    return (y.to(torch.bfloat16) if out_bf16 else y).to(D)


def _ln_inputs(rows, C, seed, offset=0.0, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    x = offset + spread * torch.randn(rows, C, generator=g)
    x[::3] = torch.randn(x[::3].shape, generator=g) * 1e-3      # rows whose variance is near eps
    gamma = 1 + 0.5 * torch.randn(C, generator=g)
    beta = 0.5 * torch.randn(C, generator=g)
    return x, gamma, beta


@pytest.mark.parametrize("C", [132, 768, 1280])
@pytest.mark.parametrize("out_bf16", [True, False])
@pytest.mark.parametrize("gelu", [False, True])
def test_layernorm_bound_holds_and_defects_fall_outside(C, out_bf16, gelu):
    eps = 1e-6
    x, gamma, beta = _ln_inputs(48, C, seed=C, offset=300.0)
    ref = gk.layernorm_rows(x, gamma, beta, eps, gelu=gelu)
    tol = gk.layernorm_rows_tol(x, gamma, beta, eps, ref, out_bf16, gelu=gelu)
    em = lambda **kw: _ln_emulate(x, gamma, beta, eps, out_bf16, gelu, **kw)  # noqa: E731
    ratio = lambda got: gk.max_ratio((got - ref).abs(), tol)  # noqa: E731
    assert ratio(em()) <= 1.0
    defects = {"one-pass variance": em(one_pass=True), "eps outside the square root": em(eps_outside=True),
               "src_map shifted by one row": em(src_shift=1)}
    if gelu and not out_bf16:
        defects["tanh GELU"] = em(tanh=True)
    for name, got in defects.items():
        assert ratio(got) > 1.0, name


def test_layernorm_reference_gathers_and_zero_pads():
    x, gamma, beta = _ln_inputs(10, 132, seed=1)
    sm = torch.tensor([3, -1, 0, 9, -1], dtype=torch.int32)
    ref = gk.layernorm_rows(x, gamma, beta, 1e-6, src_map=sm)
    assert torch.equal(ref[1], torch.zeros(132, dtype=D)) and torch.equal(ref[4], ref[1])
    assert torch.allclose(ref[0], gk.layernorm_rows(x[3:4], gamma, beta, 1e-6)[0])
    tol = gk.layernorm_rows_tol(x, gamma, beta, 1e-6, ref, True, src_map=sm)
    assert tol[1].max().item() < 1e-20


# ---------------------------------------------------------------------------------------------------- rejections
def test_row_kernels_reject_bad_arguments_before_launch():
    """Pointer alignment for every vector access, and the shapes the host arithmetic needs, are checked before any
    device work (so these addresses are never dereferenced), with a message that names what was broken."""
    from rsprompter_b200 import _lib
    L = _lib._lib
    base = 1 << 24
    I, O, G, B, CP = (base * (i + 1) for i in range(5))

    def err(st):
        return st, (L.rsp_last_error() or b"").decode()

    def ln(inp=I, in_fp32=1, out=O, out_fp32=0, g=G, b=B, cp=None):
        return err(L.rsp_layernorm(inp, in_fp32, 256, out, out_fp32, 256, g, b, None, 8, 256, 1e-6, 0, cp,
                                   256 if cp else 0, None))

    def im2col(H=8, W=8, C=8, KH=3, KW=3, stride=1, pad=1, inp=I, out=O):
        return err(L.rsp_im2col_nhwc(inp, out, 1, H, W, C, KH, KW, stride, pad, None))

    cases = [
        (ln(inp=I + 8), "in must be 16-byte"), (ln(inp=I + 4, in_fp32=0), "in must be 8-byte"),
        (ln(out=O + 4), "out must be 8-byte"), (ln(out=O + 8, out_fp32=1), "out must be 16-byte"),
        (ln(g=G + 4), "gamma / beta"), (ln(b=B + 8), "gamma / beta"), (ln(cp=CP + 4), "copy_out must be 8-byte"),
        (err(L.rsp_patchify16(I + 8, O, 1, 32, 32, None)), "img / out must be 16-byte"),
        (err(L.rsp_patchify16(I, O + 8, 1, 32, 32, None)), "img / out must be 16-byte"),
        (err(L.rsp_patchify16(I, O, 1, 0, 32, None)), "patchify: shape"),
        (err(L.rsp_patchify16(I, O, 1, 32, -16, None)), "patchify: shape"),
        (im2col(stride=0), "stride 0"), (im2col(stride=-1), "stride -1"), (im2col(KH=0), "kernel 0x3"),
        (im2col(KW=-1), "kernel 3x-1"), (im2col(pad=-1), "pad -1"),
        (im2col(H=2, W=2, KH=5, KW=5, pad=0), "larger than the padded 2x2"),
        (im2col(H=8, W=2, KH=5, KW=5, pad=1), "larger than the padded 10x4"),
        (im2col(inp=I + 8), "in / out must be 16-byte"), (im2col(out=O + 2), "in / out must be 16-byte"),
        (im2col(C=0), "im2col: shape"),
        (err(L.rsp_cast_f32_bf16(I + 8, O, 64, None)), "in must be 16-byte and out 8-byte"),
        (err(L.rsp_cast_f32_bf16(I, O + 4, 64, None)), "in must be 16-byte and out 8-byte"),
        (err(L.rsp_add_table_bf16(I + 8, G, O, 64, 16, None)), "x / table / out must be 16-byte"),
        (err(L.rsp_add_table_bf16(I, G + 4, O, 64, 16, None)), "x / table / out must be 16-byte"),
        (err(L.rsp_add_table_bf16(I, G, O + 8, 64, 16, None)), "x / table / out must be 16-byte"),
    ]
    for i, ((st, msg), want) in enumerate(cases):
        assert st != 0 and want in msg, (i, st, msg)
