"""The mask decoder's fused kernels against the kernel chains they replace, on the same bf16 inputs.

Both fused kernels keep every rounding point and the order of every sum of the chain they replace, so their outputs
must equal it byte for byte:
  * t2i_fused computes the k | v projection with the GEMM's wgmma shape and k order, rounds it where the GEMM
    epilogue rounds it ((acc + bias) + residual), and runs t2i_attention's per-head step over the keys in order;
  * i2t_fused does the same for the Qimg projection, runs i2t_attention's per-(16 rows, head) step, and sums the
    LayerNorm statistics of the out_proj in the column order of the EPI_LN_ROW GEMM epilogue."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _t2i_inputs(n, hw, tq, seed, v_residual=False):
    g = torch.Generator().manual_seed(seed)
    keys = torch.randn(n * hw, 256, generator=g).to(torch.bfloat16)
    kvw = (0.06 * torch.randn(256, 256, generator=g)).to(torch.bfloat16)
    kvb = 0.1 * torch.randn(256, generator=g)
    pe = torch.zeros(hw, 256)
    pe[:, :128] = torch.randn(hw, 128, generator=g)          # the decoder's layout: the v half is 0
    if v_residual:
        pe[:, 128:] = torch.randn(hw, 128, generator=g)
    q = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    return [t.cuda() for t in (q, keys, kvw, kvb, pe.to(torch.bfloat16))]


def _chain(q, keys, kvw, kvb, pe, hw):
    from rsprompter_b200 import _lib
    KV = _lib.gemm(keys, kvw, kvb, residual=pe, res_mod=hw)
    return _lib.t2i_attention(q, KV[:, :128], KV[:, 128:], hw)


@pytest.mark.parametrize("n,hw,tq", [
    (800, 4096, 10),    # C3: 8 images x 100 queries, 64 x 64 tokens
    (1, 4096, 10),
    (133, 1024, 10),    # not a multiple of the 132 SMs; 32 x 32 tokens
    (7, 1024, 6),
    (5, 4096, 16),
    (3, 900, 10),       # 30 x 30 tokens: a partial last tile of 4 keys
    (2, 40, 10),        # one partial tile
])
def test_t2i_fused_equals_gemm_then_attention(n, hw, tq):
    from rsprompter_b200 import _lib
    q, keys, kvw, kvb, pe = _t2i_inputs(n, hw, tq, seed=n + hw + tq)
    ref = _chain(q, keys, kvw, kvb, pe, hw)
    out = _lib.t2i_fused(q, keys, kvw, kvb, pe, hw)
    again = _lib.t2i_fused(q, keys, kvw, kvb, pe, hw)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), \
        f"max |diff| {(out.float() - ref.float()).abs().max().item()}"
    assert torch.equal(out.view(torch.int16), again.view(torch.int16))


def test_t2i_fused_residual_on_both_halves_and_strided_keys():
    from rsprompter_b200 import _lib
    n, hw, tq = 9, 1024, 10
    q, keys, kvw, kvb, pe = _t2i_inputs(n, hw, tq, seed=5, v_residual=True)
    wide = torch.zeros(n * hw, 320, device="cuda", dtype=torch.bfloat16)
    wide[:, 32:288] = keys
    strided = wide[:, 32:288]
    ref = _chain(q, keys, kvw, kvb, pe, hw)
    out = _lib.t2i_fused(q, strided, kvw, kvb, pe, hw)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


def test_t2i_fused_rejects_bad_arguments():
    from rsprompter_b200 import _lib
    q, keys, kvw, kvb, pe = _t2i_inputs(2, 1024, 10, seed=3)
    with pytest.raises(_lib.RspError):
        _lib._check(_lib._lib.rsp_t2i_fused(_lib._ptr(keys), 256, _lib._ptr(kvw), _lib._ptr(kvb), _lib._ptr(pe),
                                            _lib._ptr(q), _lib._ptr(q), 2, 17, 1024, None), "rsp_t2i_fused")
    with pytest.raises(_lib.RspError):
        _lib._check(_lib._lib.rsp_t2i_fused(_lib._ptr(keys), 100, _lib._ptr(kvw), _lib._ptr(kvb), _lib._ptr(pe),
                                            _lib._ptr(q), _lib._ptr(q), 2, 10, 1024, None), "rsp_t2i_fused")


def _i2t_inputs(n, hw, tq, seed):
    g = torch.Generator().manual_seed(seed)
    # rows with a large common offset exercise the shifted LayerNorm statistics
    keys = (torch.randn(n * hw, 256, generator=g) + 4.0 * torch.randn(n * hw, 1, generator=g)).to(torch.bfloat16)
    wq = (0.06 * torch.randn(128, 256, generator=g)).to(torch.bfloat16)
    qb = 0.1 * torch.randn(128, generator=g)
    pe_q = torch.randn(hw, 128, generator=g).to(torch.bfloat16)
    ktok = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    vtok = torch.randn(n, tq, 128, generator=g).to(torch.bfloat16)
    wo = (0.09 * torch.randn(256, 128, generator=g)).to(torch.bfloat16)
    ob = 0.1 * torch.randn(256, generator=g)
    lg = 1.0 + 0.1 * torch.randn(256, generator=g)
    lb = 0.1 * torch.randn(256, generator=g)
    return [t.cuda() for t in (keys, wq, qb, pe_q, ktok, vtok, wo, ob, lg, lb)]


def _i2t_chain(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln, hw):
    from rsprompter_b200 import _lib
    Q = _lib.gemm(keys, wq, qb, residual=pe_q, res_mod=hw)
    att = _lib.i2t_attention(Q, ktok, vtok, hw)
    return _lib.gemm(att, wo, ob, residual=keys, ln=ln)


@pytest.mark.parametrize("n,hw,tq", [
    (800, 4096, 10),    # C3
    (1, 4096, 10),
    (133, 1024, 10),    # fewer tiles per CTA in the last round than in the others
    (7, 1024, 6),
    (5, 4096, 16),
    (3, 192, 10),       # a prompt of three 64-row tiles
])
def test_i2t_fused_equals_q_gemm_attention_ln_gemm(n, hw, tq):
    from rsprompter_b200 import _lib
    keys, wq, qb, pe_q, ktok, vtok, wo, ob, lg, lb = _i2t_inputs(n, hw, tq, seed=n + hw + tq)
    ln = (lg, lb, 1e-6)
    ref = _i2t_chain(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln, hw)
    out = _lib.i2t_fused(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln, hw)
    again = _lib.i2t_fused(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln, hw)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), \
        f"max |diff| {(out.float() - ref.float()).abs().max().item()}, " \
        f"{(out != ref).sum().item()} of {out.numel()} differ"
    assert torch.equal(out.view(torch.int16), again.view(torch.int16))


def test_i2t_fused_strided_keys():
    from rsprompter_b200 import _lib
    n, hw, tq = 9, 1024, 10
    keys, wq, qb, pe_q, ktok, vtok, wo, ob, lg, lb = _i2t_inputs(n, hw, tq, seed=8)
    wide = torch.zeros(n * hw, 320, device="cuda", dtype=torch.bfloat16)
    wide[:, 64:320] = keys
    ref = _i2t_chain(keys, wq, qb, pe_q, ktok, vtok, wo, ob, (lg, lb, 1e-5), hw)
    out = _lib.i2t_fused(wide[:, 64:320], wq, qb, pe_q, ktok, vtok, wo, ob, (lg, lb, 1e-5), hw)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


def test_i2t_fused_rejects_bad_arguments():
    from rsprompter_b200 import _lib
    keys, wq, qb, pe_q, ktok, vtok, wo, ob, lg, lb = _i2t_inputs(2, 1024, 10, seed=3)
    P = _lib._ptr
    def call(ldk, tq, hw):
        return _lib._lib.rsp_i2t_fused(P(keys), ldk, P(wq), P(qb), P(pe_q), P(ktok), P(vtok), P(wo), P(ob), P(lg),
                                       P(lb), 1e-6, P(keys), 2, tq, hw, None)
    for args in ((256, 17, 1024), (100, 10, 1024), (256, 10, 1000)):
        with pytest.raises(_lib.RspError):
            _lib._check(call(*args), "rsp_i2t_fused")


@pytest.mark.parametrize("multimask", [False, True])
def test_decode_per_prompt_keys_equal_the_unfused_chain(multimask, monkeypatch):
    """The whole decode with per-prompt sources (the query head's call) gives the same bytes with the fused kernels
    as with the kernel chains they replace."""
    from rsprompter_b200 import _lib, synthetic
    from rsprompter_b200.sam_config import SamDecoderArch
    from rsprompter_b200.sam_decoder import SamMaskDecoderB200
    arch = SamDecoderArch()
    dec = SamMaskDecoderB200(arch)
    dec.load_state_dict(synthetic.mask_decoder_state_dict(arch, seed=4))
    dec = dec.cuda()
    g = torch.Generator().manual_seed(4)
    n, h = 6, 64
    src = torch.randn(n * h * h, 256, generator=g).to(torch.bfloat16).cuda()
    pos = torch.randn(h * h, 256, generator=g).cuda()
    sparse = torch.randn(n, 5, 256, generator=g).cuda()
    masks, iou = dec.decode(None, pos, sparse, (h, h), src_pair=(src, None), multimask_output=multimask)

    def unfused(q, keys, kvw, kvb, pe_kv, hw):
        return _chain(q, keys, kvw, kvb, pe_kv, hw)

    monkeypatch.setattr(_lib, "t2i_fused", unfused)
    monkeypatch.setattr(_lib, "i2t_fused", _i2t_chain)
    masks_ref, iou_ref = dec.decode(None, pos, sparse, (h, h), src_pair=(src, None), multimask_output=multimask)
    torch.cuda.synchronize()
    assert torch.equal(masks, masks_ref) and torch.equal(iou, iou_ref)
