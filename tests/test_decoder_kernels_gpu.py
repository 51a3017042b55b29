"""The mask decoder's kernels one by one against the float64 restatements of oracle/decoder_kernels.py.

Each case asserts |kernel - reference| <= tol element by element, with tol derived from the kernel's rounding
points (oracle/decoder_kernels.py, the *_tol functions):
  * a bf16 result costs 2^-8 |x| (bf16 keeps 8 significant bits, so round-to-nearest is within 2^-8 relative);
  * the bf16 probabilities P of t2i / i2t cost <= 2^-8 max|V| per head: P V is taken on rounded P, the row sum on
    the unrounded ones, so every weight is off by at most 2^-8 of itself;
  * an fp32 sum of K terms costs about K 2^-24 sum|terms| (the logits, P V over the keys, the GEMM accumulators,
    the LayerNorm statistics); a logit error ds moves a softmax-weighted mean by at most 2 ds max|V|;
  * GELU on the v2 epilogues is gelu_fast, within 4e-6 of erf GELU (checked here too); |GELU'| <= 1.13.
Where a case has an exact answer it is asserted exactly: one key (t2i HW = 1), one token (i2t Tq = 1, token
self-attention T = 1) return that key's value bit for bit.  The references run in float64 on the GPU, by torch."""
import pytest
import torch

from oracle import decoder_kernels as dk

pytestmark = pytest.mark.gpu


def _check(out, ref, tol, what):
    err = (out.to(torch.float64) - ref).abs()
    ratio = (err / tol).max().item()
    print(f"{what}: max|err| {err.max().item():.3e}  max|err|/tol {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: max |err| / tol = {ratio:.3f}, max |err| = {err.max().item():.3e}"


def _cuda(*ts):
    return [None if t is None else t.cuda() for t in ts]


@pytest.mark.parametrize("T", [1, 5, 7, 10, 16])
@pytest.mark.parametrize("heads,c", [(8, 32), (3, 16)])
def test_token_self_attention(T, heads, c):
    """The decoder's 8 heads x 32 and the ABI's c = 16 at 3 heads (N * heads not a multiple of the 4 warps of a
    block); sharp logits; per-head value offsets."""
    from rsprompter_b200 import _lib
    for n in (1, 3, 800):
        q, k, v = _cuda(*dk.token_inputs(n, T, heads, c, seed=100 * T + n))
        out = _lib.token_self_attention(q, k, v, heads)
        torch.cuda.synchronize()
        if T == 1:
            assert torch.equal(out, v)
        ref = dk.token_attention(q, k, v, heads)
        _check(out, ref, dk.token_attention_tol(q, k, v, heads, ref), f"token T={T} heads={heads} c={c} n={n}")


@pytest.mark.parametrize("hw", [1, 40, 64, 900, 1024, 2500, 4096])
@pytest.mark.parametrize("layout", ["separate", "shared"])
def test_t2i_attention(hw, layout):
    """separate: K and V two [3 hw, 128] matrices, prompt n reads block n.  shared: K and V the two halves of one
    [3 hw, 256] matrix (ldkv = 256), seven prompts over a non-monotone kv_block with repeats that includes the last
    block.  A partial last tile (hw % 64 != 0) carries the sharpest logit of a (token, head) in its last valid key."""
    from rsprompter_b200 import _lib
    shared = layout == "shared"
    kv_block = [2, 0, 2, 1, 1, 0, 2] if shared else None
    n = 7 if shared else 3
    for tq in (1, 6, 10, 16):
        q, K, V, blk = dk.t2i_inputs(n, hw, tq, 3, seed=hw + tq, kv_block=kv_block)
        q, blk = _cuda(q, blk)
        if shared:
            kv = torch.cat([K, V], dim=1).cuda()
            K, V = kv[:, :128], kv[:, 128:]
        else:
            K, V = _cuda(K, V)
        out = _lib.t2i_attention(q, K, V, hw, kv_block=blk)
        torch.cuda.synchronize()
        if hw == 1:
            rows = blk.long() if shared else torch.arange(n, device="cuda")
            assert torch.equal(out, V[rows].unsqueeze(1).expand(-1, tq, -1))
        ref = dk.t2i(q, K, V, hw, kv_block=blk)
        _check(out, ref, dk.t2i_tol(q, K, V, hw, ref, kv_block=blk), f"t2i {layout} hw={hw} tq={tq}")


@pytest.mark.parametrize("hw", [1, 100, 900, 1024, 4096])
@pytest.mark.parametrize("mapped", [False, True])
def test_i2t_attention(hw, mapped):
    """Partial 128-row tiles (hw = 100, 900), padded tokens (tq < 16) under logits far below 0, q_block maps."""
    from rsprompter_b200 import _lib
    q_block = [2, 0, 2, 1, 1, 0, 2] if mapped else None
    n = 7 if mapped else 3
    for tq in (1, 2, 10, 16):
        Q, kt, vt, qb = _cuda(*dk.i2t_inputs(n, hw, tq, 3, seed=hw + tq, q_block=q_block))
        out = _lib.i2t_attention(Q, kt, vt, hw, q_block=qb)
        torch.cuda.synchronize()
        if tq == 1:
            assert torch.equal(out.view(n, hw, 128), vt.expand(n, hw, 128))
        ref = dk.i2t(Q, kt, vt, hw, q_block=qb)
        _check(out, ref, dk.i2t_tol(Q, kt, vt, hw, ref, q_block=qb), f"i2t mapped={mapped} hw={hw} tq={tq}")


def _fused(n, hw, tq, seed):
    t = dk.fused_inputs(n, hw, tq, seed)
    return {k: (tuple(_cuda(*v[:2])) + (v[2],) if k == "ln" else v.cuda()) for k, v in t.items()}


@pytest.mark.parametrize("n,hw,tq", [(800, 4096, 10), (3, 900, 10)])
def test_t2i_fused_against_float64(n, hw, tq):
    """t2i_fused directly against float64 (the bar any re-ordering of its softmax, such as splitting a prompt's keys
    across CTAs, is held to); the operands make the k | v projection exact in fp32 (dk.fused_inputs)."""
    from rsprompter_b200 import _lib
    t = _fused(n, hw, tq, seed=n + hw)
    out = _lib.t2i_fused(t["q"], t["keys"], t["kvw"], t["kvb"], t["pe_kv"], hw)
    torch.cuda.synchronize()
    worst, worst_err = 0.0, 0.0
    for p0 in range(0, n, 100):
        p1 = min(n, p0 + 100)
        ref, tol = dk.t2i_fused_ref_tol(t["q"][p0:p1], t["keys"][p0 * hw:p1 * hw], t["kvw"], t["kvb"], t["pe_kv"], hw)
        err = (out[p0:p1].double() - ref).abs()
        worst, worst_err = max(worst, (err / tol).max().item()), max(worst_err, err.max().item())
    print(f"t2i_fused n={n} hw={hw}: max|err| {worst_err:.3e}  max|err|/tol {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("n,hw,tq", [(800, 4096, 10), (3, 192, 10)])
def test_i2t_fused_against_float64(n, hw, tq):
    from rsprompter_b200 import _lib
    t = _fused(n, hw, tq, seed=n + hw)
    out = _lib.i2t_fused(t["keys"], t["wq"], t["qb"], t["pe_q"], t["ktok"], t["vtok"], t["wo"], t["ob"], t["ln"], hw)
    torch.cuda.synchronize()
    worst, worst_err = 0.0, 0.0
    for p0 in range(0, n, 100):
        p1 = min(n, p0 + 100)
        rows = slice(p0 * hw, p1 * hw)
        ref, tol = dk.i2t_fused_ref_tol(t["keys"][rows], t["wq"], t["qb"], t["pe_q"], t["ktok"][p0:p1],
                                        t["vtok"][p0:p1], t["wo"], t["ob"], t["ln"], hw)
        err = (out[rows].double() - ref).abs()
        worst, worst_err = max(worst, (err / tol).max().item()), max(worst_err, err.max().item())
    print(f"i2t_fused n={n} hw={hw}: max|err| {worst_err:.3e}  max|err|/tol {worst:.3f}")
    assert worst <= 1.0


def test_prepare_uses_the_oracle_layouts():
    """SamMaskDecoderB200._prepare() lays the upscaler and k | v weights out as the references read them."""
    from rsprompter_b200 import synthetic
    from rsprompter_b200.sam_config import SamDecoderArch
    from rsprompter_b200.sam_decoder import SamMaskDecoderB200
    dec = SamMaskDecoderB200(SamDecoderArch())
    dec.load_state_dict(synthetic.mask_decoder_state_dict(SamDecoderArch(), seed=3))
    dec = dec.cuda()
    p = dec._prepare()
    bf = lambda t: t.detach().to(torch.bfloat16)  # noqa: E731
    assert torch.equal(p["up1_w"], bf(dk.convt_gemm_weight(dec.upscale_conv1.weight)))
    assert torch.equal(p["up2_w"], bf(dk.convt_gemm_weight(dec.upscale_conv2.weight)))
    assert torch.equal(p["up1_b"], dk.convt_gemm_bias(dec.upscale_conv1.bias).float())
    assert torch.equal(p["up2_b"], dk.convt_gemm_bias(dec.upscale_conv2.bias).float())
    a = dec.transformer.layers[0].cross_attn_token_to_image
    assert torch.equal(p["layers"][0]["t2i"]["kvw"], bf(torch.cat([a.k_proj.weight, a.v_proj.weight])))


@pytest.mark.parametrize("h,w", [(64, 64), (32, 32), (30, 30), (24, 40)])
@pytest.mark.parametrize("ldo", [256, 260])
def test_upscale1_ln_gelu(h, w, ldo):
    """epi_mode 2 (upscale_conv1 + LayerNorm2d + GELU), compared after reassembling the (pixel, tap) rows into
    (N, 64, 2h, 2w).  30 x 30: prompt boundaries inside 128-row tiles; 24 x 40: y / x swaps show.  ldo 256: TMA
    store of a contiguous output; 260: the direct store path."""
    from rsprompter_b200 import _lib
    n = 3
    t = dk.upscale_inputs(n, h, w, seed=h * w + ldo)
    W1, b1 = dk.convt_gemm_weight(t["w1"]).to(torch.bfloat16), dk.convt_gemm_bias(t["b1"])
    keys, W1, b1, g, b = _cuda(t["keys"], W1, b1, t["gamma"], t["beta"])
    buf = torch.full((n * h * w, ldo), float("nan"), device="cuda", dtype=torch.bfloat16)
    out = _lib.gemm(keys, W1, b1, out=buf[:, :256], ln64_gelu=(g, b, 1e-6))
    torch.cuda.synchronize()
    assert buf[:, 256:].isnan().all()
    ref = dk.upscale1_ln_gelu(keys, W1, b1, g, b, 1e-6, h, w)
    _check(dk.up1_rows_to_image(out.double(), h, w), ref, dk.upscale1_tol(keys, W1, b1, g, 1e-6, h, w, ref),
           f"upscale1 {h}x{w} ldo={ldo}")


@pytest.mark.parametrize("h,w", [(64, 64), (30, 30), (40, 25)])
@pytest.mark.parametrize("P", [1, 7, 133])
def test_upscale2_hyper(h, w, P):
    """epi_mode 3 (upscale_conv2 + GELU + hypernetwork product) on 64 x 64, 30 x 30 and 40 x 25 (odd grid_w).  The
    one-hot hyper case pins the pixel placement Y = 4y + 2ty1 + ty2, X = 4x + 2tx1 + tx2."""
    from rsprompter_b200 import _lib
    for one_hot in (False, True):
        up1, W2, b2, hyper = _cuda(*dk.upscale2_inputs(P, h, w, seed=P + h + w, one_hot=one_hot))
        out = _lib.gemm_upscale_mask(up1, W2, b2, hyper, h, w)
        torch.cuda.synchronize()
        ref = dk.upscale2_hyper(up1, W2, b2, hyper, h, w)
        _check(out, ref, dk.upscale2_tol(up1, W2, b2, hyper, h, w), f"upscale2 {h}x{w} P={P} one_hot={one_hot}")


def test_gelu_fast_error_bound():
    """sm90.cuh gelu_fast (the v2 GEMM epilogues' GELU): within 4e-6 + 4 ulp of float64 erf GELU on [-9, 9],
    exactly 0 below -9 and exactly x above 9.  Driven through a GEMM with A = 0, so each output is GELU(bias);
    the SIMT GEMM (gelu_erf) gives the same values within the same bound."""
    from rsprompter_b200 import _lib
    x = torch.cat([torch.linspace(-12, 12, 48001),    # + 9 = an even column count: the v2 kernel takes fp32 output
                   torch.tensor([9.0, -9.0, 20.0, -20.0, 1e4, -1e4, 1e30, -1e30, 0.0])]).float()
    a = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(x.numel(), 64, device="cuda", dtype=torch.bfloat16)
    xb = x.cuda()
    fast = _lib.gemm(a, w, xb, act="gelu", out_dtype=torch.float32)
    simt = _lib.gemm(a, w, xb, act="gelu", out_dtype=torch.float32, simt=True)
    torch.cuda.synchronize()
    assert torch.equal(fast, fast[:1].expand_as(fast))
    ref = dk.gelu_erf64(x).cuda()
    ulp = (torch.nextafter(ref.float().abs(), torch.tensor(float("inf"), device="cuda")) - ref.float().abs()).double()
    inside = x.abs().cuda() <= 9
    for y, what in ((fast[0], "gelu_fast"), (simt[0], "gelu_erf")):
        err = (y.double() - ref).abs()
        print(f"{what}: max|err| on [-9, 9] {err[inside].max().item():.3e}")
        assert (err[inside] <= 4e-6 + 4 * ulp[inside]).all(), what
        assert torch.equal(y[xb < -9], torch.zeros_like(y[xb < -9])), what
        assert torch.equal(y[xb > 9], xb[xb > 9]), what
