"""The encoder's row kernels (rowops.cu, and patchify16_u8 in records.cu) against float64 or CPU torch:
  * layernorm within oracle/gemm_kernels.layernorm_rows_tol for every dtype pair and MAXV, strided rows, large-mean
    rows, GELU and the window gather; padding rows exact zeros, copy_out exactly bf16(x), every other byte untouched;
  * patchify16, patchify16_u8, im2col_nhwc, cast_bf16 and nhwc_to_nchw byte for byte."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_kernels as gk

pytestmark = pytest.mark.gpu

BF16, FP32 = torch.bfloat16, torch.float32


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _ln_inputs(rows, C, in_dtype, seed, ld_in):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g) * torch.exp2(torch.randint(-3, 3, (rows, 1), generator=g).float())
    x[1::2] += 300.0                                                    # mean >> spread
    x[::5] *= 1e-3                                                      # variance near eps
    buf = torch.full((rows, ld_in), float("nan"), dtype=in_dtype)
    buf[:, :C] = x.to(in_dtype)
    gamma = 1 + 0.5 * torch.randn(C, generator=g)
    beta = 0.5 * torch.randn(C, generator=g)
    return buf.cuda()[:, :C], gamma.cuda(), beta.cuda()


def _ln_check(x, gamma, beta, eps, out_dtype, gelu, src_map=None, copy=False, label=""):
    from rsprompter_b200 import _lib
    rows_out = x.shape[0] if src_map is None else src_map.numel()
    C = x.shape[1]
    ob = torch.full((rows_out + 2, C + 8), float("nan"), dtype=out_dtype, device="cuda")
    sent = ob.clone()
    cp = cps = None
    if copy:
        cp = torch.full((x.shape[0] + 1, C + 4), float("nan"), dtype=BF16, device="cuda")
        cps = cp.clone()
    _lib.layernorm(x, gamma, beta, eps, out=ob[:rows_out, :C], src_map=src_map, gelu=gelu,
                   copy_out=None if cp is None else cp[:x.shape[0], :C])
    torch.cuda.synchronize()
    ref = gk.layernorm_rows(x, gamma, beta, eps, src_map=src_map, gelu=gelu)
    tol = gk.layernorm_rows_tol(x, gamma, beta, eps, ref, out_dtype == BF16, src_map=src_map, gelu=gelu)
    got = ob[:rows_out, :C]
    ratio = gk.max_ratio((got.double() - ref).abs(), tol)
    print(f"layernorm {label} C={C} {x.dtype}->{out_dtype} gelu={gelu}: max|err|/tol = {ratio:.3f}")
    assert ratio <= 1.0
    outside = torch.ones_like(ob, dtype=torch.bool)
    outside[:rows_out, :C] = False
    assert torch.equal(_bits(ob)[outside], _bits(sent)[outside])
    if src_map is not None:
        pad = src_map < 0
        assert torch.equal(_bits(got[pad]), torch.zeros_like(_bits(got[pad])))       # +0.0 exactly
    if copy:
        read = torch.zeros(x.shape[0] + 1, dtype=torch.bool, device="cuda")
        read[src_map[src_map >= 0].long()] = True
        want = cps.clone()
        want[:x.shape[0], :C][read[:x.shape[0]]] = x[read[:x.shape[0]]].to(BF16)
        assert torch.equal(_bits(cp), _bits(want))


@pytest.mark.parametrize("C", [4, 132, 256, 260, 768, 1024, 1280])
@pytest.mark.parametrize("in_dtype,out_dtype", [(FP32, BF16), (FP32, FP32), (BF16, BF16), (BF16, FP32)])
@pytest.mark.parametrize("gelu", [False, True])
def test_layernorm(C, in_dtype, out_dtype, gelu):
    x, gamma, beta = _ln_inputs(300, C, in_dtype, seed=C, ld_in=C + 4)
    _ln_check(x, gamma, beta, 1e-6, out_dtype, gelu)


@pytest.mark.parametrize("grid,window,C", [(20, 14, 768), (16, 14, 1280), (9, 4, 256)])
def test_layernorm_window_gather_and_copy_out(grid, window, C):
    from rsprompter_b200.sam_encoder import window_maps
    x, gamma, beta = _ln_inputs(2 * grid * grid, C, FP32, seed=grid, ld_in=C)
    x = x.contiguous()
    wmap, _ = window_maps(2, grid, window, torch.device("cuda"))
    assert (wmap < 0).any()
    _ln_check(x, gamma, beta, 1e-6, BF16, False, src_map=wmap, copy=True, label="window")


def test_patchify16():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(0)
    img = torch.randn(2, 3, 64, 96, generator=g) * 100
    got = _lib.patchify16(img.cuda())
    want = img.view(2, 3, 4, 16, 6, 16).permute(0, 2, 4, 1, 3, 5).reshape(-1, 768).to(BF16)
    assert torch.equal(_bits(got.cpu()), _bits(want))


@pytest.mark.parametrize("hwc", [False, True])
@pytest.mark.parametrize("swap_rb", [False, True])
def test_patchify16_u8(hwc, swap_rb):
    """(u - mean) / std in fp32 with one rounding each (__fsub_rn / __fdiv_rn), then RNE to bf16: torch's bytes."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(1)
    B, H, W = 2, 48, 80
    u8 = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    mean, std = (123.675, 116.28, 103.53), (58.395, 57.12, 57.375)
    dev = u8.permute(0, 2, 3, 1).contiguous().cuda().permute(0, 3, 1, 2) if hwc else u8.cuda()
    got = _lib.patchify16_u8(dev, mean, std, swap_rb)
    x = u8.float()[:, [2, 1, 0]] if swap_rb else u8.float()
    x = (x - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    want = x.view(B, 3, H // 16, 16, W // 16, 16).permute(0, 2, 4, 1, 3, 5).reshape(-1, 768).to(BF16)
    assert torch.equal(_bits(got.cpu()), _bits(want))


@pytest.mark.parametrize("k", [1, 3, 5])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("pad", [0, 1, 2])
def test_im2col_nhwc(k, stride, pad):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(k * 10 + stride + pad)
    B, H, W, C = 2, 13, 10, 24
    x = torch.randn(B, H, W, C, generator=g).to(BF16)
    got = _lib.im2col_nhwc(x.cuda(), k, k, stride, pad)
    cols = F.unfold(x.permute(0, 3, 1, 2).double(), k, padding=pad, stride=stride)       # [B, C k k, L]
    L = cols.shape[-1]
    want = cols.view(B, C, k * k, L).permute(0, 3, 2, 1).reshape(B * L, k * k * C).to(BF16)
    assert torch.equal(_bits(got.cpu()), _bits(want))


def test_cast_bf16_rounding_edges():
    from rsprompter_b200 import _lib
    one = 1.0
    special = torch.tensor([
        one + 2 ** -8, one + 3 * 2 ** -8, -(one + 2 ** -8), -(one + 3 * 2 ** -8),      # ties: to even
        one + 2 ** -8 + 2 ** -20, 2.0 ** -126 * 1.5, 1e-40, -1e-39, 1.4e-45, -1.4e-45, 2.0 ** -133 * 3,  # subnormals
        3.3961e38, -3.3961e38, 3.4028235e38, 3.3895e38,                                  # to +-inf, max bf16
        float("inf"), float("-inf"), float("nan"), 0.0, -0.0,
    ], dtype=FP32)
    g = torch.Generator().manual_seed(2)
    rand = torch.randn(4000, generator=g) * torch.exp2(torch.randint(-140, 128, (4000,), generator=g).float())
    ties = (torch.randint(-2 ** 15, 2 ** 15, (1000,), generator=g).int() << 16 | 0x8000).view(FP32)
    x = torch.cat([special, rand, ties])
    x = torch.cat([x, x.new_zeros((-x.numel()) % 4)])
    got = _lib.cast_bf16(x.cuda()).cpu()
    want = x.to(BF16)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(_bits(got)[~nan], _bits(want)[~nan])


@pytest.mark.parametrize("dtype", [FP32, BF16])
def test_nhwc_to_nchw(dtype):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 7, 9, 45, generator=g).to(dtype)
    got = _lib.nhwc_to_nchw(x.cuda()).cpu()
    assert torch.equal(_bits(got), _bits(x.permute(0, 3, 1, 2).float().contiguous()))
