"""Kernel-level parity on the GPU, through the C ABI (ctypes), against the CPU oracle / plain
fp32 torch math on the same seeded inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _rel_err(got, ref):
    return (got.float().cpu() - ref.float().cpu()).abs().max().item() / max(ref.abs().max().item(), 1e-6)


@pytest.mark.parametrize("M,N,K,act,res,out_dtype", [
    (300, 768, 768, None, False, torch.bfloat16),
    (1000, 2304, 768, None, False, torch.bfloat16),
    (1000, 3072, 768, "gelu", False, torch.bfloat16),
    (1000, 768, 3072, None, True, torch.float32),
    (777, 40, 256, "relu", False, torch.float32),
    (64, 256, 2048, None, True, torch.float32),
    # odd N: rows of 4-byte (fp32) and 2-byte (bf16) alignment take the epilogue's scalar path
    (800, 11, 256, None, False, torch.float32),
    (300, 11, 256, "relu", True, torch.bfloat16),
])
def test_gemm_matches_fp32_reference(M, N, K, act, res, out_dtype):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(M + N + K)
    a = _bf(torch.randn(M, K, generator=g))
    w = _bf(torch.randn(N, K, generator=g) * K ** -0.5)
    b = torch.randn(N, generator=g)
    r = torch.randn(M, N, generator=g) if res else None
    ref = a.float() @ w.float().t() + b
    if act == "gelu":
        ref = torch.nn.functional.gelu(ref)
    elif act == "relu":
        ref = torch.relu(ref)
    if res:
        ref = ref + r
    out = _lib.gemm(a.cuda(), w.cuda(), b.cuda(), act=act, residual=r.cuda() if res else None,
                    out_dtype=out_dtype)
    torch.cuda.synchronize()
    tol = 1e-2 if out_dtype == torch.bfloat16 else 2e-5 * K ** 0.5 + 1e-4
    assert _rel_err(out, ref) < tol


def test_gemm_row_map_and_broadcast_residual():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(3)
    M, N, K, rows = 500, 256, 128, 400
    a = _bf(torch.randn(M, K, generator=g))
    w = _bf(torch.randn(N, K, generator=g) * 0.1)
    perm = torch.randperm(M, generator=g)
    row_map = torch.full((M,), -1, dtype=torch.int32)
    row_map[perm[:rows]] = torch.arange(rows, dtype=torch.int32)
    pos = torch.randn(100, N, generator=g)
    out = torch.zeros(rows, N, device="cuda")
    _lib.gemm(a.cuda(), w.cuda(), None, out=out, residual=pos.cuda(), res_mod=100, row_map=row_map.cuda())
    torch.cuda.synchronize()
    full = a.float() @ w.float().t()
    ref = torch.zeros(rows, N)
    for m in range(M):
        d = row_map[m].item()
        if d >= 0:
            ref[d] = full[m] + pos[d % 100]
    assert _rel_err(out, ref) < 1e-4


def test_gemm_simt_agrees_with_tensor_core_path():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(4)
    a = _bf(torch.randn(130, 256, generator=g)).cuda()
    w = _bf(torch.randn(96, 256, generator=g) * 0.1).cuda()
    b = torch.randn(96, generator=g).cuda()
    x = _lib.gemm(a, w, b, out_dtype=torch.float32)
    y = _lib.gemm(a, w, b, out_dtype=torch.float32, simt=True)
    torch.cuda.synchronize()
    assert _rel_err(x, y.cpu()) < 1e-5


@pytest.mark.parametrize("S,n_seq,H,hd", [(14, 5, 3, 64), (14, 5, 2, 80), (64, 1, 2, 64), (64, 1, 2, 80)])
def test_vit_attention_matches_oracle(S, n_seq, H, hd):
    from oracle import restate
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(S + hd)
    T, D = S * S, H * hd
    qkv = _bf(torch.randn(n_seq * T, 3 * D, generator=g))
    rh = _bf(torch.randn(2 * S - 1, hd, generator=g) * 0.2)
    rw = _bf(torch.randn(2 * S - 1, hd, generator=g) * 0.2)
    x = qkv.float().reshape(n_seq, T, 3, H, hd).permute(2, 0, 3, 1, 4).reshape(3, n_seq * H, T, hd)
    ref = restate.vit_attention_core(x[0], x[1], x[2], rh.float(), rw.float(), S)
    ref = ref.reshape(n_seq, H, T, hd).permute(0, 2, 1, 3).reshape(n_seq * T, D)
    out = _lib.vit_attention(qkv.cuda(), rh.cuda(), rw.cuda(), n_seq, S, H, hd)
    simt = _lib.vit_attention(qkv.cuda(), rh.cuda(), rw.cuda(), n_seq, S, H, hd, simt=True)
    torch.cuda.synchronize()
    assert _rel_err(simt, ref) < 1e-2      # bf16 output rounding only
    assert _rel_err(out, ref) < 1.5e-2     # + bf16 P, fp16 rel-pos row term


def test_layernorm_with_window_gather():
    from rsprompter_b200 import _lib
    from rsprompter_b200.sam_encoder import window_maps
    from oracle import restate
    g = torch.Generator().manual_seed(9)
    B, grid, C = 2, 64, 768
    x = torch.randn(B, grid, grid, C, generator=g)
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ref = torch.nn.functional.layer_norm(x, (C,), w, b, 1e-6)
    ref_win, _ = restate.window_partition(ref, 14)
    wmap, n_win = window_maps(B, grid, 14, torch.device("cuda"))
    assert n_win == 25
    out = _lib.layernorm(x.reshape(-1, C).cuda(), w.cuda(), b.cuda(), 1e-6, src_map=wmap)
    torch.cuda.synchronize()
    assert out.shape == (B * 25 * 196, C)
    assert _rel_err(out, ref_win.reshape(-1, C)) < 1e-2
    out32 = _lib.layernorm(x.reshape(-1, C).cuda(), w.cuda(), b.cuda(), 1e-6, out_dtype=torch.float32)
    assert _rel_err(out32, ref.reshape(-1, C)) < 1e-5


def test_patchify_im2col_transpose():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(10)
    img = torch.randn(2, 3, 64, 96, generator=g)
    w = torch.randn(32, 3, 16, 16, generator=g)
    ref = torch.nn.functional.conv2d(_bf(img).float(), w, stride=16).permute(0, 2, 3, 1).reshape(-1, 32)
    p = _lib.patchify16(img.cuda())
    got = p.float().cpu() @ w.reshape(32, -1).t()
    assert _rel_err(got, ref) < 1e-5
    x = _bf(torch.randn(2, 10, 12, 16, generator=g))
    wc = torch.randn(24, 16, 3, 3, generator=g)
    for stride in (1, 2):
        ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wc, stride=stride, padding=1)
        col = _lib.im2col_nhwc(x.cuda(), 3, 3, stride, 1)
        got = col.float().cpu() @ wc.permute(0, 2, 3, 1).reshape(24, -1).t()
        assert _rel_err(got, ref.permute(0, 2, 3, 1).reshape(-1, 24)) < 1e-5
    t = _lib.nhwc_to_nchw(x.cuda())
    torch.cuda.synchronize()
    assert torch.equal(t.cpu(), x.float().permute(0, 3, 1, 2))


def test_wrong_device_raises():
    from rsprompter_b200 import _lib
    with pytest.raises(_lib.RspError):
        _lib.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


@pytest.mark.parametrize("B,H,W,C,N", [(2, 64, 64, 64, 96), (1, 256, 256, 64, 32), (3, 8, 8, 128, 256),
                                       (2, 16, 16, 64, 24), (5, 4, 4, 64, 64), (1, 128, 128, 256, 256)])
def test_conv3x3_implicit_gemm(B, H, W, C, N):
    """rsp_conv3x3_nhwc_bf16 (4-D TMA taps, zero-filled halo) against F.conv2d on the same bf16 values."""
    import torch.nn.functional as F
    from rsprompter_b200 import _lib
    from rsprompter_b200.necks import prep_conv
    assert _lib.conv3x3_ok(B, H, W, C)
    g = torch.Generator().manual_seed(B * 1000 + H)
    x = torch.randn(B, C, H, W, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, C, 3, 3, generator=g) / (3 * C ** 0.5)).to(torch.bfloat16)
    b = torch.randn(N, generator=g)
    res = torch.randn(B * H * W, N, generator=g)
    wg, bg = prep_conv(w.float(), b)
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    ref = F.conv2d(x.float(), w.float(), b, padding=1)
    out = _lib.conv3x3_nhwc(xh, wg.cuda(), bg.cuda()).float().cpu().view(B, H, W, N).permute(0, 3, 1, 2)
    assert (out - ref).abs().max().item() < 3e-2
    ref2 = F.relu(ref).permute(0, 2, 3, 1).reshape(B * H * W, N) + res
    out2 = _lib.conv3x3_nhwc(xh, wg.cuda(), bg.cuda(), act="relu", residual=res.cuda(), out_dtype=torch.float32).cpu()
    assert (out2 - ref2).abs().max().item() < 2e-2


def test_conv3x3_geometry_gate():
    from rsprompter_b200 import _lib
    assert not _lib.conv3x3_ok(1, 64, 64, 32)        # C % 64
    assert not _lib.conv3x3_ok(1, 14, 14, 256)       # 14 x 14 RoI maps do not tile into 128-pixel boxes
    assert not _lib.conv3x3_ok(1, 48, 48, 64)
    assert _lib.conv3x3_ok(8, 256, 256, 256) and _lib.conv3x3_ok(8, 16, 16, 128)


@pytest.mark.parametrize("M,offset,res_dtype,block", [
    pytest.param(4096, 0.0, torch.bfloat16, None, id="4096-0.0"),
    pytest.param(4096, 300.0, torch.bfloat16, None, id="4096-300.0"),
    pytest.param(37, 300.0, torch.bfloat16, None, id="37-300.0"),
    # prompts mapped onto their image's residual rows (res_block_map): 32-row TMA residual slabs ...
    pytest.param(5 * 1024, 300.0, torch.bfloat16, (1024, [2, 0, 1, 2, 0]), id="map1024"),
    pytest.param(3 * 4096, 0.0, torch.bfloat16, (4096, [1, 1, 0]), id="map4096"),
    # ... and per-row residual reads when a block is not a whole number of slabs
    pytest.param(4 * 900, 300.0, torch.bfloat16, (900, [1, 0, 1, 2]), id="map900"),
    # fp32 residual and output: the decoder's token path
    pytest.param(8000, 0.0, torch.float32, None, id="fp32res-8000"),
    pytest.param(70, 300.0, torch.float32, None, id="fp32res-70"),
    # no residual, fp32 output: the decoder's first ln1
    pytest.param(5600, 0.0, None, None, id="nores-5600"),
])
def test_gemm_fused_row_layernorm_large_mean(M, offset, res_dtype, block):
    """LN(acc + bias + residual) fused into the GEMM epilogue (mask decoder layer_norm4 / token norms, HF:346-347) on
    rows whose mean dwarfs their spread: the statistics must not lose the variance to E[x^2] - E[x]^2 cancellation.
    Checked against float64 (oracle/decoder_kernels.ln_row) within the bound of the epilogue's rounding points
    (ln_row_tol: fp32 accumulation and statistics, bf16 output 2^-8 |y|), and within 4e-2 absolute."""
    from oracle import decoder_kernels as dk
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(7)
    K, N = 128, 256
    a = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.1
    rows, bmap = block if block else (M, None)
    res = None if res_dtype is None else (torch.randn((max(bmap) + 1) * rows if bmap else M, N, generator=g) +
                                          offset).to(res_dtype)
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g), 0.1 * torch.randn(N, generator=g)
    rm = {} if bmap is None else dict(res_block_map=torch.tensor(bmap, dtype=torch.int32), res_block_rows=rows)
    ref = dk.ln_row(a, w, bias, res, gamma, beta, 1e-6, **rm)
    if res_dtype in (torch.float32, None):
        out_dtypes = (torch.float32,)
    else:
        out_dtypes = (torch.bfloat16, torch.float32) if M < 128 else (torch.bfloat16,)
    for out_dtype in out_dtypes:
        out = _lib.gemm(a.cuda(), w.cuda(), bias.cuda(), residual=None if res is None else res.cuda(),
                        ln=(gamma.cuda(), beta.cuda(), 1e-6),
                        out_dtype=out_dtype, **{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in rm.items()})
        torch.cuda.synchronize()
        err = (out.double().cpu() - ref).abs()
        tol = dk.ln_row_tol(a, w, bias, res, gamma, beta, 1e-6, ref, out_bf16=out_dtype == torch.bfloat16, **rm)
        print(f"ln_row M={M} offset={offset} res={res_dtype} block={rows if bmap else None} out={out_dtype}: "
              f"max|err| {err.max().item():.3e}  max|err|/tol {(err / tol).max().item():.3f}")
        assert err.max().item() < 4e-2 and (err <= tol).all(), (M, offset, out_dtype, (err / tol).max().item())
