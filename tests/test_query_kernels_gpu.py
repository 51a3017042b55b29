"""The query head's standalone kernels one by one against the float64 references of oracle/query_kernels.py.

Each case asserts |kernel - reference| <= tol element by element, with tol derived from the kernel's rounding points
(the *_tol functions; tests/test_query_kernels_cpu.py shows each bound rejects a plausible defect), and prints
max|err| and max|err|/tol.  Inputs are bf16 where the kernel reads bf16, so the reference sees the kernel's values.
The references run in float64 on the GPU, by torch."""
import pytest
import torch

from oracle import query_kernels as qk

pytestmark = pytest.mark.gpu

LEVELS = {1: [(6, 10)], 2: [(12, 20), (1, 1)], 3: [(6, 10), (12, 20), (3, 5)], 4: [(6, 10), (12, 20), (3, 5), (1, 1)]}


def _check(out, ref, tol, what):
    err = (out.to(torch.float64) - ref).abs()
    ratio = (err / tol).max().item()
    print(f"{what}: max|err| {err.max().item():.3e}  max|err|/tol {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: max |err| / tol = {ratio:.3f}, max |err| = {err.max().item():.3e}"


@pytest.mark.parametrize("hd", [16, 32])
@pytest.mark.parametrize("L", [1, 2, 3, 4])
@pytest.mark.parametrize("P", [1, 4, 5])
def test_ms_deform_attn_sample(hd, L, P):
    """Non-square levels and a 1 x 1 level, B = 2, NQ not a multiple of the 128-thread block, ld_ow past the row;
    samples fully and half outside a map, on integer and half-integer pixels and exactly at -1 and W / H; logits
    N(0, 2), spread above 80, and all equal."""
    from rsprompter_b200 import _lib
    shapes = LEVELS[L]
    for logits in ("normal", "spread", "equal"):
        value, ow = qk.deform_inputs(shapes, P, hd, 2, seed=100 * L + 10 * P + hd, logits=logits)
        value, ow = value.cuda(), ow.cuda()
        out = _lib.ms_deform_attn_sample(value, ow, shapes, P)
        torch.cuda.synchronize()
        ref = qk.ms_deform_core(value, ow, shapes, P)
        _check(out, ref, qk.ms_deform_tol(value, ow, shapes, P, ref), f"ms_deform hd={hd} L={L} P={P} {logits}")


def _grouped_case(a, w, N, mgr, wgr, row_map, out_rows, out_dtype, what):
    """Run gemm_grouped into a NaN-filled [out_rows + 3, N + 8] buffer (ldo = N + 8) and check the mapped rows
    against float64, and that the 3 unmapped rows and the 8 columns past N still hold NaN."""
    from rsprompter_b200 import _lib
    buf = torch.full((out_rows + 3, N + 8), float("nan"), device="cuda", dtype=out_dtype)
    _lib.gemm_grouped(a, w, buf[:, :N], N, mgr, wgr, row_map=row_map)
    torch.cuda.synchronize()
    assert buf[:, N:].isnan().all() and buf[out_rows:].isnan().all(), f"{what}: wrote outside the mapped block"
    ref = qk.grouped_gemm(a, w, N, mgr, wgr, row_map, out_rows=out_rows)
    assert not ref.isnan().any()
    tol = qk.grouped_gemm_tol(a, w, N, mgr, wgr, ref, row_map, out_bf16=out_dtype == torch.bfloat16)
    _check(buf[:out_rows, :N], ref, tol, what)


@pytest.mark.parametrize("hw_l", [144, 576, 2304, 256, 1024, 4096, 400, 1600, 6400])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_gemm_grouped_query_head(hw_l, out_dtype):
    """The query head's per-level mask logits: me_pad [8 x 128, 256] (100 queries + 28 padding rows per image, the
    padding rows not 0), one [hw_l, 256] feature block per image (hw_l of 768, 1024 and 1280 inputs; N % 128 != 0
    for 144, 400, 1600), no slack rows after the last image's block, image weights 10^(b % 4 - 1) apart."""
    me, mf, back = qk.grouped_inputs(8, 100, hw_l, seed=hw_l)
    _grouped_case(me.cuda(), mf.cuda(), hw_l, 128, hw_l, back.cuda(), 800, out_dtype,
                  f"gemm_grouped N={hw_l} {str(out_dtype)[6:]}")


def test_gemm_grouped_attention_shape():
    """vit_attention_generic's P V: m_group_rows = T = 2304 (48 x 48 tokens), N = w_group_rows = hd = 80, K = T, and
    the head scatter map (stacked row (h, t) -> row t H + h), four heads whose V differ by orders of magnitude."""
    T, H, hd = 2304, 4, 80
    g = torch.Generator().manual_seed(7)
    P = torch.rand(H * T, T, generator=g).pow(8)
    P = (P / P.sum(-1, keepdim=True)).to(torch.bfloat16)
    vt = (torch.randn(H * hd, T, generator=g) * (10.0 ** (torch.arange(H) - 1.0)).repeat_interleave(hd).view(-1, 1))
    t, h = torch.arange(T, dtype=torch.int32), torch.arange(H, dtype=torch.int32)
    rmap = (t.view(1, T) * H + h.view(H, 1)).reshape(-1).contiguous()
    _grouped_case(P.cuda(), vt.to(torch.bfloat16).cuda(), hd, T, hd, rmap.cuda(), T * H, torch.bfloat16,
                  "gemm_grouped attention P V")


@pytest.mark.parametrize("hw,want_pe,mma", [((64, 64), False, True), ((48, 48), False, True),
                                            ((16, 16), False, True), ((40, 40), False, False),
                                            ((64, 2), False, False), ((64, 64), True, False)])
def test_mask_embed_src(hw, want_pe, mma):
    """Both kernels, reached by shape: the mma kernel takes h w % 128 == 0 and w % 4 == 0 without src_pe; the fp32
    kernel takes 40 x 40 (h w % 128 != 0), 64 x 2 (w % 4 != 0) and every src_pe call.  3 images x 5 prompts; mask
    logits up to +-20, exact-zero and constant 4 x 4 patches.  The fp32 kernel is held to its own, tighter bound."""
    from rsprompter_b200 import _lib
    N, npi = 15, 5
    weights = [w.cuda() for w in qk.mask_embed_weights(seed=hw[0] + hw[1])]
    mpp, emb, pos = [t.cuda() for t in qk.mask_embed_inputs(N, hw, npi, seed=hw[0] * hw[1])]
    src, src_pe = _lib.mask_embed_src(mpp, weights, emb, pos, npi, hw, want_pe=want_pe)
    torch.cuda.synchronize()
    ref, ref_pe = qk.sam_mask_embed_src(mpp, weights, emb, pos, npi, hw)
    what = f"mask_embed_src {hw[0]}x{hw[1]} {'mma' if mma else 'fp32'}"
    _check(src, ref, qk.mask_embed_src_tol(mpp, weights, ref, mma=mma), what)
    if want_pe:
        _check(src_pe, ref_pe, qk.mask_embed_src_tol(mpp, weights, ref_pe, mma=mma, pos=pos), what + " src_pe")
