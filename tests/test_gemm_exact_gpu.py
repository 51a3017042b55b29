"""The standard epilogue of the wgmma GEMM (rsp_gemm_bf16 epi_mode 0 and the implicit 3x3 convolution) byte for byte
against float64, on every path of gemm_v2.cu.

The operands come from oracle/gemm_kernels.exact_operands: small integers times powers of two, on which the fp32
accumulator is exact in any summation order.  The kernel's bytes are then defined: fp32(acc + bias), the activation,
fp32(. + residual), round to nearest even where the output is bf16 (gemm_expect).  GELU is the one inexact step;
its bytes must lie between the roundings of GELU(erf) -/+ GELU_FAST_ERR.

Every output lives in a NaN-filled buffer with a wider row stride and extra rows: the written block must hold exactly
the expected bytes and every other byte the sentinel, destination rows a row map drops included.  Cases that exist to
reach a path assert the instantiation that ran (gemm_bf16_wgmma_v2_kernel<BN, EPI>), so a change to a gate cannot
move them off it silently."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_kernels as gk

pytestmark = pytest.mark.gpu

BF16, FP32 = torch.bfloat16, torch.float32
WIDE = "gemm_bf16_wgmma_v2_kernel<256, 7>"
SPLIT = {32: "gemm_bf16_wgmma_v2_kernel<32, 0>", 64: "gemm_bf16_wgmma_v2_kernel<64, 0>",
         128: "gemm_bf16_wgmma_v2_kernel<128, 0>"}


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "gemm_bf16_wgmma" in e.name}


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


class Out:
    """A [rows, N] output view at element `offset` of a NaN-filled flat buffer, row stride ldo, `extra` spare rows."""

    def __init__(self, rows, N, dtype, ldo=None, offset=0, extra=3):
        self.rows, self.N, self.ldo, self.offset = rows, N, ldo or (N + 8), offset
        self.buf = torch.full(((rows + extra) * self.ldo + offset,), float("nan"), dtype=dtype, device="cuda")
        self.sentinel = self.buf.clone()
        self.view = self._block(self.buf)

    def _block(self, flat):
        return flat[self.offset:self.offset + self.rows * self.ldo].view(self.rows, self.ldo)[:, :self.N]

    def _expected(self, val):
        e = self.sentinel.clone()
        blk = self._block(e)
        keep = ~torch.isnan(val)
        blk[keep] = val[keep]
        return e

    def mismatches(self, lo, hi) -> int:
        """Elements of the whole buffer that differ from the expected bytes (lo is hi) or lie outside [lo, hi]."""
        elo = self._expected(lo)
        if lo is hi:
            return int((_bits(self.buf) != _bits(elo)).sum().item())
        ehi = self._expected(hi)
        sent = torch.isnan(elo)
        bad = sent & (_bits(self.buf) != _bits(self.sentinel))
        bad |= ~sent & ((self.buf < elo) | (self.buf > ehi) | torch.isnan(self.buf))
        return int(bad.sum().item())


def _gemm_exact(name, M, N, K, *, seed, act=None, bias=True, residual=None, res_rows=None, ldr=None, res_mod=0,
                res_block_map=None, res_block_rows=0, row_map=None, out_rows=None, out_dtype=BF16, ldo=None,
                out_offset=0, bias_offset=0, lda=None, ldw=None, kernel=None, repeat=1):
    """One exact-operand call into a sentinel buffer; asserts zero mismatches (and the instantiation when given)."""
    from rsprompter_b200 import _lib
    a, w, b, r = gk.exact_operands(M, N, K, seed, bias=bias, residual=residual, res_rows=res_rows, res_cols=ldr,
                                   lda=lda, ldw=ldw)
    if b is not None and bias_offset:
        b = torch.cat([b.new_zeros(bias_offset), b])[bias_offset:]
    if r is not None and ldr:
        r = r[:, :N]
    rows = out_rows or M
    out = Out(rows, N, out_dtype, ldo=ldo, offset=out_offset)
    rmap = dict(res_mod=res_mod, res_block_map=res_block_map, res_block_rows=res_block_rows, row_map=row_map)
    call = lambda: _lib.gemm(a, w, b, out=out.view, act=act, residual=r, **rmap)  # noqa: E731
    names = _kernels(call)
    lo, hi = gk.gemm_expect(a, w, b, act, r, out_dtype, out_rows=rows, **rmap)
    bad = out.mismatches(lo, hi)
    first = out.buf.clone()
    for _ in range(repeat - 1):
        out.buf.copy_(out.sentinel)
        call()
        torch.cuda.synchronize()
        assert torch.equal(_bits(out.buf), _bits(first)), f"{name}: repeated call changed the bytes"
    ran = sorted(n.split("(")[0].replace("void ", "").replace("rsp::v2::", "") for n in names)
    print(f"{name}: M={M} N={N} K={K} mismatches={bad} kernel={ran}")
    assert bad == 0, name
    if kernel is not None:
        assert any(kernel in n for n in names), (name, names)


# ---------------------------------------------------------------------------------------------------- tile tails
@pytest.mark.parametrize("N", [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 257])
@pytest.mark.parametrize("M", [1, 127, 129, 1000])
def test_tile_tails(M, N):
    bn = 32 if N <= 32 else 64 if N <= 64 else 128
    _gemm_exact("tail", M, N, 136, seed=M * 1000 + N, act="relu", out_dtype=FP32 if M == 129 else BF16,
                residual="grid" if M == 1000 else None, kernel=SPLIT[bn])


# ---------------------------------------------------------------------------------------------------- double-buffered
@pytest.mark.parametrize("N", [12, 32, 48])
@pytest.mark.parametrize("out_dtype", [BF16, FP32])
@pytest.mark.parametrize("residual", [False, True])
def test_double_buffered_accumulator_many_tiles_per_cta(N, out_dtype, residual):
    """BN <= 64 double-buffers the accumulator tile: 547 tiles over at most 132 CTAs alternate buffers and phases."""
    res = ("grid" if out_dtype == FP32 else "bf16") if residual else None
    _gemm_exact("double-buffered", 70001, N, 256, seed=N, out_dtype=out_dtype, residual=res,
                kernel=SPLIT[32 if N <= 32 else 64])


# ---------------------------------------------------------------------------------------------------- K tails
@pytest.mark.parametrize("K", [8, 72, 200, 1288])
def test_k_tails_with_nan_padded_operands(K):
    """lda, ldw > K with NaN in the padding columns: a tensor map that read past K would put NaN in the output."""
    pad = K + 8
    _gemm_exact("k-tail", 300, 96, K, seed=K, lda=pad, ldw=pad, out_dtype=FP32, residual="grid", kernel=SPLIT[128])
    _gemm_exact("k-tail", 300, 96, K, seed=K + 1, lda=pad, ldw=pad, act="gelu")


# ---------------------------------------------------------------------------------------------------- schedules
@pytest.mark.parametrize("M,N,K,act", [(39200, 3840, 1280, None), (32768, 5120, 1280, "gelu")])
def test_wide_schedule(M, N, K, act):
    """ViT-H qkv and lin1: 128 x 256 tiles with the epilogue in registers, twice, byte-identical."""
    _gemm_exact("wide", M, N, K, seed=N, act=act, kernel=WIDE, repeat=2)


@pytest.mark.parametrize("case", ["vitb_qkv", "proj", "lin2", "patch_embed"])
def test_split_schedule_tma_out_and_residual(case):
    if case == "vitb_qkv":
        _gemm_exact(case, 9800, 2304, 768, seed=1, kernel=SPLIT[128])
    elif case == "proj":
        _gemm_exact(case, 9800, 768, 768, seed=2, residual="grid", out_dtype=FP32, kernel=SPLIT[128])
    elif case == "lin2":
        _gemm_exact(case, 9800, 768, 3072, seed=3, residual="grid", out_dtype=FP32, kernel=SPLIT[128])
    else:
        _gemm_exact(case, 8192, 768, 768, seed=4, residual="grid", res_rows=4096, res_mod=4096, out_dtype=FP32,
                    kernel=SPLIT[128])


def _row_map(M, rows, seed):
    """Destination rows in reverse order with every 7th source row dropped: rows - 1 - m, or -1."""
    rm = torch.arange(rows - 1, rows - 1 - M, -1, dtype=torch.int32)
    rm[torch.arange(M) % 7 == 3] = -1
    return rm.cuda()


@pytest.mark.parametrize("case", ["res_mod_100", "res_mod_100_gelu", "bf16_res_fp32_out", "block_map_1024",
                                  "block_map_900", "row_map_res_mod"])
def test_split_schedule_scatter(case):
    if case.startswith("res_mod_100"):
        _gemm_exact(case, 1000, 256, 320, seed=5, residual="grid", res_rows=100, res_mod=100, out_dtype=FP32,
                    act="gelu" if case.endswith("gelu") else None, kernel=SPLIT[128])
    elif case == "bf16_res_fp32_out":
        _gemm_exact(case, 1000, 192, 320, seed=6, residual="bf16", out_dtype=FP32, act="relu", kernel=SPLIT[128])
    elif case == "block_map_1024":
        bm = torch.tensor([2, 0, 1, 2], dtype=torch.int32, device="cuda")
        _gemm_exact(case, 4096, 256, 256, seed=7, residual="grid", res_rows=3 * 1024, res_block_map=bm,
                    res_block_rows=1024, out_dtype=FP32, kernel=SPLIT[128])
    elif case == "block_map_900":
        bm = torch.tensor([1, 1, 0, 2], dtype=torch.int32, device="cuda")
        _gemm_exact(case, 3600, 256, 256, seed=8, residual="grid", res_rows=3 * 900, res_block_map=bm,
                    res_block_rows=900, out_dtype=FP32, kernel=SPLIT[128])
    else:
        _gemm_exact(case, 1000, 160, 200, seed=9, residual="grid", res_rows=64, res_mod=64, act="relu",
                    row_map=_row_map(1000, 1100, 9), out_rows=1100, kernel=SPLIT[128])


@pytest.mark.parametrize("case", ["odd_n_odd_ldo", "out_odd_offset", "bias_4_byte_offset"])
def test_scalar_rows(case):
    """Rows the epilogue cannot move 8 bytes at a time, each with a residual and a row map."""
    rm = _row_map(500, 520, 10)
    if case == "odd_n_odd_ldo":
        _gemm_exact(case, 500, 77, 200, seed=10, residual="grid", res_rows=520, ldr=79, row_map=rm, out_rows=520,
                    ldo=83, out_dtype=FP32, kernel=SPLIT[128])
    elif case == "out_odd_offset":
        _gemm_exact(case, 500, 64, 200, seed=11, residual="bf16", res_rows=520, row_map=rm, out_rows=520,
                    out_offset=1, act="relu", kernel=SPLIT[64])
    else:
        _gemm_exact(case, 500, 128, 200, seed=12, residual="grid", res_rows=520, row_map=rm, out_rows=520,
                    bias_offset=1, out_dtype=FP32, kernel=SPLIT[128])


@pytest.mark.parametrize("out_dtype", [BF16, FP32])
def test_arbitrary_fp32_residual_rounds_once(out_dtype):
    """Any fp32 residual: acc + bias is exact, so the residual add is the one IEEE rounding (and then the bf16 one)."""
    _gemm_exact("fp32 residual", 2048, 256, 512, seed=13, residual="fp32", out_dtype=out_dtype, act="relu")


# ---------------------------------------------------------------------------------------------------- implicit conv
def _conv_operands(B, H, W, C, N, seed):
    x, w, b, _ = gk.exact_operands(B * H * W, N, 9 * C, seed)
    x = x[:, :C].contiguous().view(B, H, W, C)
    # im2col of the float64 conv (F.unfold: (c, ky, kx) columns) in the kernel's (ky, kx, c) order
    cols = F.unfold(x.permute(0, 3, 1, 2).double(), 3, padding=1).view(B, C, 9, H * W)
    cols = cols.permute(0, 3, 2, 1).reshape(B * H * W, 9 * C).to(BF16)
    return x, w, b, cols


@pytest.mark.parametrize("B,H,W,C", [(3, 8, 8, 64), (2, 16, 16, 64), (1, 64, 64, 256), (2, 128, 128, 64),
                                     (1, 256, 256, 64)])
@pytest.mark.parametrize("N", [24, 96, 256])
@pytest.mark.parametrize("variant", ["relu_bf16", "residual_fp32"])
def test_implicit_conv3x3(B, H, W, C, N, variant):
    from rsprompter_b200 import _lib
    assert _lib.conv3x3_ok(B, H, W, C)
    x, w, b, cols = _conv_operands(B, H, W, C, N, seed=B * H * C + N)
    M = B * H * W
    act, out_dtype = ("relu", BF16) if variant == "relu_bf16" else (None, FP32)
    r = gk.exact_operands(M, N, 8, seed=N, residual="grid")[3] if variant == "residual_fp32" else None
    out = Out(M, N, out_dtype)
    _lib._check(_lib._lib.rsp_conv3x3_nhwc_bf16(
        x.data_ptr(), B, H, W, C, w.data_ptr(), w.stride(0), out.view.data_ptr(), out.ldo, N, b.data_ptr(),
        None if r is None else r.data_ptr(), 0 if r is None else r.stride(0), 1, _lib.ACT[act],
        int(out_dtype == FP32), _lib._stream()), "rsp_conv3x3_nhwc_bf16")
    torch.cuda.synchronize()
    lo, hi = gk.gemm_expect(cols, w, b, act, r, out_dtype)
    bad = out.mismatches(lo, hi)
    print(f"conv3x3 {(B, H, W, C)} N={N} {variant}: mismatches={bad}")
    assert bad == 0


def test_rejected_conv_geometry_falls_back_to_im2col_exactly():
    """A geometry conv3x3_ok rejects (W = 20: a 128-pixel tile is no box) takes im2col + gemm, as the neck does."""
    from rsprompter_b200 import _lib
    B, H, W, C, N = 2, 20, 20, 64, 96
    assert not _lib.conv3x3_ok(B, H, W, C)
    x, w, b, cols = _conv_operands(B, H, W, C, N, seed=20)
    got = _lib.im2col_nhwc(x, 3, 3, 1, 1)
    assert torch.equal(_bits(got), _bits(cols))
    out = Out(B * H * W, N, BF16)
    _lib.gemm(got, w, b, out=out.view, act="relu")
    lo, hi = gk.gemm_expect(cols, w, b, "relu", None, BF16)
    assert out.mismatches(lo, hi) == 0


# ---------------------------------------------------------------------------------------------------- real operands
def _real(M, N, K, seed, residual=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, generator=g, device="cuda").to(BF16)
    w = (torch.randn(N, K, generator=g, device="cuda") * K ** -0.5).to(BF16)
    b = torch.randn(N, generator=g, device="cuda")
    r = torch.randn(M, N, generator=g, device="cuda") if residual else None
    return a, w, b, r


@pytest.mark.parametrize("M,N,K,act,residual,out_dtype,kernel", [
    (32768, 3840, 1280, None, False, BF16, WIDE),               # ViT-H qkv
    (9800, 768, 3072, None, True, FP32, SPLIT[128]),            # ViT-B lin2 + residual
    (8192, 64, 768, "gelu", False, BF16, SPLIT[64]),
    (131072, 32, 256, None, False, FP32, SPLIT[32]),            # RPN head, batch 2 over a 256 x 256 level
])
def test_real_operands_within_bound(M, N, K, act, residual, out_dtype, kernel):
    from rsprompter_b200 import _lib
    a, w, b, r = _real(M, N, K, seed=M + N, residual=residual)
    res = {}
    names = _kernels(lambda: res.setdefault("out", _lib.gemm(a, w, b, act=act, residual=r, out_dtype=out_dtype)))
    assert any(kernel in n for n in names), names
    ref = gk.gemm_std(a, w, b, act, r)
    tol = gk.gemm_std_tol(a, w, b, act, r, ref, out_dtype == BF16)
    ratio = gk.max_ratio((res["out"].double() - ref).abs(), tol)
    print(f"real {kernel} M={M} N={N} K={K} act={act}: max|err|/tol = {ratio:.3f}")
    assert ratio <= 1.0
