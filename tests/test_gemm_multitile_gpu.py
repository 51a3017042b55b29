"""Persistent GEMM with many tiles per CTA: at M = 33 000 (not a multiple of 128) every CTA runs tens of tiles, so the
hand-off of the accumulator tile from the MMA warpgroups to the epilogue warps goes through every buffer and phase
state.  Reference: fp32 torch on the GPU with TF32 off, same tolerances as test_gemm_matches_fp32_reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M = 33000


@pytest.fixture(autouse=True)
def _no_tf32():
    mm, cd = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cd


def _inputs(m, n, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(m, k, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(n, k, generator=g, device="cuda") * k ** -0.5).to(torch.bfloat16)
    b = torch.randn(n, generator=g, device="cuda")
    return a, w, b, g


def _rel_err(got, ref):
    return (got.float() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)


def _tol(out_dtype, k):
    return 1e-2 if out_dtype == torch.bfloat16 else 2e-5 * k ** 0.5 + 1e-4


@pytest.mark.parametrize("N,K,act,res", [
    (3840, 1280, None, False),     # qkv: bias -> bf16
    (1280, 1280, "gelu", False),
    (3840, 5120, "gelu", False),
    (1280, 1280, None, True),      # proj: bias + fp32 residual -> fp32
    (1280, 5120, None, True),      # lin2
])
def test_gemm_many_tiles_per_cta(N, K, act, res):
    from rsprompter_b200 import _lib
    a, w, b, g = _inputs(M, N, K, N + K)
    r = torch.randn(M, N, generator=g, device="cuda") if res else None
    out_dtype = torch.float32 if res else torch.bfloat16
    out = _lib.gemm(a, w, b, act=act, residual=r, out_dtype=out_dtype)
    ref = a.float() @ w.float().t() + b
    if act == "gelu":
        ref = torch.nn.functional.gelu(ref)
    if res:
        ref = ref + r
    torch.cuda.synchronize()
    assert _rel_err(out, ref) < _tol(out_dtype, K)


def test_gemm_many_tiles_broadcast_residual():
    """res_mod: residual row = output row % 4096 (absolute position embedding added to every image)."""
    from rsprompter_b200 import _lib
    N, K, P = 1280, 1280, 4096
    a, w, b, g = _inputs(M, N, K, 11)
    pos = torch.randn(P, N, generator=g, device="cuda")
    out = _lib.gemm(a, w, b, residual=pos, res_mod=P, out_dtype=torch.float32)
    rows = torch.arange(M, device="cuda") % P
    ref = a.float() @ w.float().t() + b + pos[rows]
    torch.cuda.synchronize()
    assert _rel_err(out, ref) < _tol(torch.float32, K)


def test_gemm_many_tiles_row_map_scatter():
    """row_map: reversed destination rows with every 7th row dropped (the scatter epilogue)."""
    from rsprompter_b200 import _lib
    N, K = 1280, 1280
    a, w, b, _ = _inputs(M, N, K, 12)
    src = torch.arange(M, device="cuda")
    keep = src % 7 != 3
    rows = int(keep.sum().item())
    row_map = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    row_map[keep] = torch.arange(rows - 1, -1, -1, dtype=torch.int32, device="cuda")
    out = torch.zeros(rows, N, device="cuda")
    _lib.gemm(a, w, b, out=out, row_map=row_map)
    full = a.float() @ w.float().t() + b
    ref = torch.zeros(rows, N, device="cuda")
    ref[row_map[keep].long()] = full[keep]
    torch.cuda.synchronize()
    assert _rel_err(out, ref) < _tol(torch.float32, K)


def test_conv3x3_many_tiles_per_cta():
    """Implicit-GEMM 3x3 conv with 2 x 128 x 128 pixels x 256 channels out = 512 tiles (> 3 per CTA on 132 SMs)."""
    import torch.nn.functional as F
    from rsprompter_b200 import _lib
    from rsprompter_b200.necks import prep_conv
    B, H, W, C, N = 2, 128, 128, 64, 256
    assert _lib.conv3x3_ok(B, H, W, C)
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(B, C, H, W, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, C, 3, 3, generator=g, device="cuda") / (3 * C ** 0.5)).to(torch.bfloat16)
    b = torch.randn(N, generator=g, device="cuda")
    res = torch.randn(B * H * W, N, generator=g, device="cuda")
    wg, bg = prep_conv(w.float().cpu(), b.cpu())
    xh = x.permute(0, 2, 3, 1).contiguous()
    out = _lib.conv3x3_nhwc(xh, wg.cuda(), bg.cuda(), act="relu", residual=res, out_dtype=torch.float32)
    ref = F.relu(F.conv2d(x.float(), w.float(), b, padding=1)).permute(0, 2, 3, 1).reshape(B * H * W, N) + res
    torch.cuda.synchronize()
    assert _rel_err(out, ref) < _tol(torch.float32, 9 * C)
