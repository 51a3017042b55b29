"""The float64 references of the mask decoder's kernels (oracle/decoder_kernels.py), checked without a GPU:
  * pinned to the fp32 restatement (oracle/restate.py): the attention cores against _sam_attention's core, the
    upscalers against mask_decoder's upscaling lines (which also pins the ConvTranspose -> GEMM-column layout);
  * bug distance: on every adversarial input of tests/test_decoder_kernels_gpu.py, a plausible kernel bug, restated
    on the reference, lands more than 10x that test's tolerance away from the right answer, so the GPU test can
    fail on it;
  * the fused GEMM epilogues reject pointers their vector accesses cannot use, before anything is launched."""
import pytest
import torch
import torch.nn.functional as F

from oracle import decoder_kernels as dk
from oracle import restate

FAR = 10.0


def _identity_attention(q, k, v, heads):
    """restate._sam_attention with identity projections: its softmax(q k^T / sqrt(c)) v core, fp32."""
    C = q.shape[-1]
    eye, zero = torch.eye(C), torch.zeros(C)
    sd = {f"{p}_proj.{s}": (eye if s == "weight" else zero) for p in ("q", "k", "v", "out") for s in ("weight", "bias")}
    return restate._sam_attention(sd, "", q.float(), k.float(), v.float(), heads)


def _close(ref64, fp32, scale):
    err = (ref64 - fp32.double()).abs().max().item()
    assert err <= 1e-5 * scale, (err, scale)


@pytest.mark.parametrize("heads,c", [(8, 32), (3, 16)])
def test_token_attention_matches_restate(heads, c):
    q, k, v = dk.token_inputs(3, 7, heads, c, seed=1)
    ref = dk.token_attention(q, k, v, heads)
    _close(ref, _identity_attention(q, k, v, heads), v.float().abs().max().item())


def test_t2i_and_i2t_match_restate():
    q, K, V, blk = dk.t2i_inputs(5, 40, 10, 3, seed=2, kv_block=[2, 0, 2, 1, 0], shared=True)
    ref = dk.t2i(q, K, V, 40, kv_block=blk)
    rows = lambda t: t.reshape(3, 40, 128)[blk.long()]  # noqa: E731
    _close(ref, _identity_attention(q, rows(K), rows(V), 8), 20.0)
    Q, kt, vt, qb = dk.i2t_inputs(5, 100, 10, 3, seed=3, q_block=[1, 1, 0, 2, 0])
    ref = dk.i2t(Q, kt, vt, 100, q_block=qb)
    exp = _identity_attention(Q.reshape(3, 100, 128)[qb.long()], kt, vt, 8).reshape(-1, 128)
    _close(ref, exp, 10.0)


def test_upscalers_match_restate_mask_decoder():
    n, h, w = 2, 3, 5
    t = dk.upscale_inputs(n, h, w, seed=4)
    img = t["keys"].float().view(n, h, w, 256).permute(0, 3, 1, 2)
    # mask_decoder's upscaling lines (restate.mask_decoder)
    up = F.conv_transpose2d(img, t["w1"], t["b1"], stride=2)
    up = F.gelu(restate.layer_norm_channels_first(up, t["gamma"], t["beta"], 1e-6))
    ref1 = dk.upscale1_ln_gelu(t["keys"], dk.convt_gemm_weight(t["w1"]), dk.convt_gemm_bias(t["b1"]), t["gamma"],
                               t["beta"], 1e-6, h, w)
    _close(ref1, up, 4.0)
    up1_rows = dk.image_to_up1_rows(up).to(torch.bfloat16)
    up_b = dk.up1_rows_to_image(up1_rows.float().reshape(-1, 256), h, w)   # the epi_mode 2 rows are the same bytes
    up2 = F.gelu(F.conv_transpose2d(up_b, t["w2"], t["b2"], stride=2))
    masks = (t["hyper"].unsqueeze(1) @ up2.reshape(n, 32, -1)).reshape(n, 4 * h, 4 * w)
    ref2 = dk.upscale2_hyper(up1_rows, dk.convt_gemm_weight(t["w2"]), dk.convt_gemm_bias(t["b2"]), t["hyper"], h, w)
    _close(ref2, masks, 10.0)
    assert torch.equal(up_b, up.to(torch.bfloat16).float())


# ---------------------------------------------------------------------------------------------------- bug distance
def _far(bug, ref, tol):
    r = dk.max_ratio((bug - ref).abs(), tol)
    assert r > FAR, f"the bug variant is only {r:.1f} x the tolerance away"


@pytest.mark.parametrize("T", [5, 16])
@pytest.mark.parametrize("heads,c", [(8, 32), (3, 16)])
def test_token_attention_bugs_are_far(T, heads, c):
    q, k, v = dk.token_inputs(3, T, heads, c, seed=T + heads)
    ref = dk.token_attention(q, k, v, heads)
    tol = dk.token_attention_tol(q, k, v, heads, ref)
    _far(dk._core(q.double() * c ** -0.5, k, v, heads), ref, tol)               # scale 1/c instead of 1/sqrt(c)
    perm = torch.arange(heads).roll(1).repeat_interleave(c) * c + torch.arange(c).repeat(heads)
    _far(dk.token_attention(q, k, v[..., perm], heads), ref, tol)               # another head's values


def _pad_clamped(X, blocks, hw):
    """Each block's rows padded to whole 64-row tiles with copies of its last row (what the unfused kernel stages)."""
    Xb = X.reshape(blocks, hw, -1)
    pad = -hw % 64
    return torch.cat([Xb, Xb[:, -1:].expand(-1, pad, -1)], dim=1).reshape(-1, X.shape[-1]), hw + pad


@pytest.mark.parametrize("hw", [40, 900, 2500])
@pytest.mark.parametrize("tq", [1, 10, 16])
def test_t2i_bugs_are_far(hw, tq):
    kv_block = [2, 0, 2, 1, 1, 0, 2]
    q, K, V, blk = dk.t2i_inputs(7, hw, tq, 3, seed=hw + tq, kv_block=kv_block, shared=True)
    ref = dk.t2i(q, K, V, hw, kv_block=blk)
    tol = dk.t2i_tol(q, K, V, hw, ref, kv_block=blk)
    Kp, hwp = _pad_clamped(K, 3, hw)
    Vp, _ = _pad_clamped(V, 3, hw)
    _far(dk.t2i(q, Kp, Vp, hwp, kv_block=blk), ref, tol)                      # clamped rows past HW counted
    _far(dk.t2i(q, K, dk.swap_heads(V), hw, kv_block=blk), ref, tol)          # heads swapped
    _far(dk.t2i(q, K, V, hw, kv_block=torch.arange(7, dtype=torch.int32) % 3), ref, tol)   # identity block map


@pytest.mark.parametrize("hw", [100, 900])
@pytest.mark.parametrize("tq", [1, 2, 10])
def test_i2t_bugs_are_far(hw, tq):
    q_block = [2, 0, 2, 1, 1, 0, 2]
    Q, kt, vt, qb = dk.i2t_inputs(7, hw, tq, 3, seed=hw + tq, q_block=q_block)
    ref = dk.i2t(Q, kt, vt, hw, q_block=qb)
    tol = dk.i2t_tol(Q, kt, vt, hw, ref, q_block=qb)
    pad = lambda t: torch.cat([t, torch.zeros(7, 16 - tq, 128, dtype=t.dtype)], dim=1)  # noqa: E731
    _far(dk.i2t(Q, pad(kt), pad(vt), hw, q_block=qb), ref, tol)               # padded tokens counted
    _far(dk.i2t(Q, kt, dk.swap_heads(vt), hw, q_block=qb), ref, tol)          # heads swapped
    if tq > 1:   # with one token every image row's answer is that token's value, whichever rows are read
        _far(dk.i2t(Q, kt, vt, hw, q_block=torch.arange(7, dtype=torch.int32) % 3), ref, tol)  # identity block map


@pytest.mark.parametrize("rows,bmap,res_fp32", [(900, [1, 0, 1, 2], False), (1024, [2, 0, 1, 2, 0], False)])
def test_ln_row_block_map_bug_is_far(rows, bmap, res_fp32):
    m = len(bmap) * rows
    a, w, bias, res, gamma, beta = dk.ln_row_inputs(m, 300.0, (max(bmap) + 1) * rows, res_fp32, seed=rows)
    rm = dict(res_block_map=torch.tensor(bmap, dtype=torch.int32), res_block_rows=rows)
    ref = dk.ln_row(a, w, bias, res, gamma, beta, 1e-6, **rm)
    tol = dk.ln_row_tol(a, w, bias, res, gamma, beta, 1e-6, ref, out_bf16=True, **rm)
    ident = dict(res_block_map=torch.arange(len(bmap), dtype=torch.int32) % (max(bmap) + 1), res_block_rows=rows)
    _far(dk.ln_row(a, w, bias, res, gamma, beta, 1e-6, **ident), ref, tol)     # residual of block n, not map[n]


@pytest.mark.parametrize("h,w", [(30, 30), (24, 40)])
def test_upscale1_tap_swap_is_far(h, w):
    t = dk.upscale_inputs(2, h, w, seed=h * w)
    W1, b1 = dk.convt_gemm_weight(t["w1"]).to(torch.bfloat16), dk.convt_gemm_bias(t["b1"])
    ref = dk.upscale1_ln_gelu(t["keys"], W1, b1, t["gamma"], t["beta"], 1e-6, h, w)
    tol = dk.upscale1_tol(t["keys"], W1, b1, t["gamma"], 1e-6, h, w, ref)
    sw = torch.tensor([0, 2, 1, 3]).repeat_interleave(64) * 64 + torch.arange(64).repeat(4)
    _far(dk.upscale1_ln_gelu(t["keys"], W1[sw], b1[sw], t["gamma"], t["beta"], 1e-6, h, w), ref, tol)   # ty <-> tx


@pytest.mark.parametrize("h,w,one_hot", [(30, 30, False), (40, 25, False), (30, 30, True)])
def test_upscale2_bugs_are_far(h, w, one_hot):
    up1, W2, b2, hyper = dk.upscale2_inputs(7, h, w, seed=h + w, one_hot=one_hot)
    ref = dk.upscale2_hyper(up1, W2, b2, hyper, h, w)
    tol = dk.upscale2_tol(up1, W2, b2, hyper, h, w)
    taps = ref.view(7, h, 2, 2, w, 2, 2).transpose(2, 3).transpose(5, 6).reshape(ref.shape)    # tap1 <-> tap2
    _far(taps, ref, tol)
    _far(ref.view(7, h, 2, 2, w, 2, 2).transpose(2, 5).reshape(ref.shape), ref, tol)          # ty1 <-> tx1
    _far(dk.upscale2_hyper(up1, W2, b2, hyper, h, w, approximate="tanh"), ref, tol)             # tanh GELU


# ---------------------------------------------------------------------------------------------------- alignment
def test_gemm_epilogue_shape_and_alignment_rejected_before_launch():
    """Every alignment the fused epilogues' vector accesses need, and the column count of epi_mode 2, is checked on
    the host: a call that breaks one returns RSP_ERR_INVALID before any device work (so these addresses are never
    dereferenced), with a message that names what was broken."""
    from rsprompter_b200 import _lib
    base = 1 << 24
    A, W, O, R, B, G, E, H, MO = (base * (i + 1) for i in range(9))

    def ex(epi, out=O, res=None, bias=B, g=G, e=E, hyper=None, mask=None, N=256, ldo=256, grid=(0, 0), res_fp32=0,
           out_fp32=0):
        M = 4 * grid[0] * grid[1] if epi == 3 else 256
        K = 64 if epi == 3 else 256
        st = _lib._lib.rsp_gemm_bf16(A, K, W, K, out, ldo, M, N, K, bias, res, 256 if res else 0, res_fp32, 0,
                                     None, 0, out_fp32, epi, g, e, 1e-6, None, 0, hyper, mask, grid[0], grid[1],
                                     None)
        return st, (_lib._lib.rsp_last_error() or b"").decode()

    cases = [
        # epi 1: out, residual, bias, gamma, beta all move 16 bytes at a time (both row-LN epilogues)
        (ex(1, out=O + 8, res=R), "alignment"), (ex(1, res=R + 8), "alignment"), (ex(1, res=R, bias=B + 4), "alignment"),
        (ex(1, res=R, g=G + 8), "alignment"), (ex(1, res=R, e=E + 4), "alignment"),
        (ex(1, out=O + 8, res=R, res_fp32=1, out_fp32=1), "alignment"),
        # epi 2: float4 bias / gamma / beta, out 8-byte aligned ...
        (ex(2, bias=B + 4), "alignment"), (ex(2, g=G + 8), "alignment"), (ex(2, e=E + 4), "alignment"),
        (ex(2, out=O + 2), "alignment"),
        # ... and N % 128 == 0
        (ex(2, out=O + 8, N=64), "N %"), (ex(2, N=64, ldo=260), "N %"),
        # epi 3: float4 hyper and bias, float2 mask stores
        (ex(3, out=None, N=128, hyper=H + 4, mask=MO, grid=(4, 6)), "alignment"),
        (ex(3, out=None, N=128, hyper=H, mask=MO + 4, grid=(4, 5)), "alignment"),
        (ex(3, out=None, N=128, hyper=H + 8, mask=MO, grid=(4, 5)), "alignment"),
        (ex(3, out=None, N=128, bias=B + 4, hyper=H, mask=MO, grid=(4, 6)), "alignment"),
    ]
    for i, ((st, msg), want) in enumerate(cases):
        assert st != 0 and want in msg, (i, st, msg)
