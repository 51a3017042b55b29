"""The 128 x 256 standard-epilogue schedule of the wgmma GEMM (accumulators kept in registers through bias, activation
and bf16 rounding) against the 128 x 128 split schedule and an fp32 torch reference with TF32 off.

The split schedule's bytes come from the same call with an output whose row stride is not a multiple of 16 bytes: such
an output cannot leave through TMA, so gemm_bf16_v2 keeps it on 128 x 128 tiles (checked by kernel name below).  The
two schedules run the same k16 wgmma sequence in the same k order and the same epilogue arithmetic, so their outputs
must be equal bit for bit, not merely close."""
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDE = "gemm_bf16_wgmma_v2_kernel<256, 7>"
SPLIT = "gemm_bf16_wgmma_v2_kernel<128, 0>"


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
    return a, w, b


def _split_out(m, n):
    """[m, n] bf16 view with a row stride of n + 4 elements (not 16-byte aligned): not TMA-eligible."""
    return torch.empty(m, n + 4, device="cuda", dtype=torch.bfloat16)[:, :n]


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "gemm_bf16_wgmma" in e.name}


def _ran(names, kernel):
    return any(kernel in n for n in names)


CASES = [
    # M, N, K, bias, act
    (39200, 3840, 1280, True, None),     # ViT-H qkv, windowed (M ragged against 128)
    (32768, 3840, 1280, True, None),     # ViT-H qkv, global
    (32768, 5120, 1280, True, "gelu"),   # ViT-H lin1
    (39200, 5120, 1280, True, "gelu"),
    (33000, 2304, 1024, False, None),    # no bias, ragged M
    (70000, 1024, 1024, True, "relu"),
    (280000, 256, 1024, True, "gelu"),   # N = 256: one n-block
]


@pytest.mark.parametrize("M,N,K,bias,act", CASES)
def test_wide_matches_split_and_fp32(M, N, K, bias, act):
    from rsprompter_b200 import _lib
    a, w, b = _inputs(M, N, K, M + N + K)
    b = b if bias else None
    res = {}
    names = _kernels(lambda: res.setdefault("wide", _lib.gemm(a, w, b, act=act)))
    assert _ran(names, WIDE), names
    wide = res["wide"]
    split = _lib.gemm(a, w, b, act=act, out=_split_out(M, N))
    torch.cuda.synchronize()
    assert torch.equal(wide, split)
    ref = a.float() @ w.float().t()
    if b is not None:
        ref = ref + b
    if act == "gelu":
        ref = torch.nn.functional.gelu(ref)
    elif act == "relu":
        ref = torch.relu(ref)
    assert (wide.float() - ref).abs().max().item() / ref.abs().max().item() < 1e-2


def test_encoder_shapes_take_the_wide_schedule():
    from rsprompter_b200 import _lib
    a, w, b = _inputs(39200, 3840, 1280, 1)
    names = _kernels(lambda: _lib.gemm(a, w, b))
    assert _ran(names, WIDE) and not _ran(names, SPLIT), names
    names = _kernels(lambda: _lib.gemm(a, w, b, out=_split_out(39200, 3840)))
    assert _ran(names, SPLIT) and not _ran(names, WIDE), names


def test_wide_is_deterministic():
    from rsprompter_b200 import _lib
    a, w, b = _inputs(32768, 5120, 1280, 2)
    x = _lib.gemm(a, w, b, act="gelu")
    y = _lib.gemm(a, w, b, act="gelu")
    torch.cuda.synchronize()
    assert torch.equal(x, y)


def test_few_tiles_stay_on_split_schedule():
    """Fewer 128 x 256 tiles than SMs: the split schedule's twice as many 128 x 128 tiles spread over more SMs."""
    from rsprompter_b200 import _lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m = 128 * (sms // 2 - 1)   # (sms / 2 - 1) m-blocks x 2 n-blocks of 256 < sms tiles
    a, w, b = _inputs(m, 512, 1280, 3)
    names = _kernels(lambda: _lib.gemm(a, w, b))
    assert _ran(names, SPLIT) and not _ran(names, WIDE), names
    out = _lib.gemm(a, w, b)
    ref = a.float() @ w.float().t() + b
    assert (out.float() - ref).abs().max().item() / ref.abs().max().item() < 1e-2


@pytest.mark.parametrize("case", ["residual", "fp32_out", "row_map", "n_not_256", "short_k"])
def test_calls_outside_the_gate_take_the_split_schedule(case):
    from rsprompter_b200 import _lib
    M = 65536   # enough tiles for the wide schedule: only the named property keeps the call off it
    N = 1408 if case == "n_not_256" else 1536   # 1408 = 11 x 128
    K = 256 if case == "short_k" else 1280
    a, w, b = _inputs(M, N, K, 4)
    kw = {}
    if case == "residual":
        kw = dict(residual=torch.randn(M, N, device="cuda"), out_dtype=torch.float32)
    elif case == "fp32_out":
        kw = dict(out_dtype=torch.float32)
    elif case == "row_map":
        kw = dict(row_map=torch.arange(M - 1, -1, -1, device="cuda", dtype=torch.int32))
    names = _kernels(lambda: _lib.gemm(a, w, b, **kw))
    assert _ran(names, SPLIT) and not _ran(names, WIDE), names
