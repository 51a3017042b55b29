"""The float64 references and bounds of the ViT encoder's attention kernels (oracle/encoder_attention.py), checked
without a GPU:
  * pinned to transformers' SamVisionAttention run in float64 (whose softmax is fp32) and to restate's fp32 core;
  * window_maps is exactly window_partition as a gather map and window_unpartition (crop included) as a scatter map;
  * the bounds are not too tight: a CPU emulation of each path's rounding points (fp32 logits, ex2 in fp32, fp16 P and
    V and the per-tile rescale for the flash kernel; fp32 per-key online softmax for the SIMT kernel; fp32 scores, a
    normalised bf16 P and a bf16 P V for the three-pass path) stays within its path's bound on every builder input;
  * the bounds are not too loose: each plausible bug, restated on the reference or on the emulation, lands more than
    FAR = 10x the bound away on the inputs tests/test_encoder_attention_gpu.py runs."""
import math

import pytest
import torch

from oracle import encoder_attention as ea
from oracle import restate

FAR = 10.0
F32 = torch.float32
LOG2E = 1.4426950408889634
# the few-tile shapes of the GPU test: (n_seq, H) = (1, 2) at every (S, hd)
FEW = dict(n_seq=1, H=2)


# ---------------------------------------------------------------------------------------------------- emulations
def _split(qkv, n_seq, S, H, hd):
    """[n_seq*T, 3*H*hd] -> q, k, v [n_seq*H, T, hd] (same dtype)."""
    T = S * S
    x = qkv.reshape(n_seq, T, 3, H, hd).permute(2, 0, 3, 1, 4).reshape(3, n_seq * H, T, hd)
    return x[0], x[1], x[2]


def _merge(o, n_seq, S, H, hd):
    T = S * S
    return o.reshape(n_seq, H, T, hd).permute(0, 2, 1, 3).reshape(n_seq * T, H * hd)


def _fma(a, b, c):
    """fp32 fmaf(a, b, c): the product is exact in float64, the sum rounds once more (below U24^2)."""
    return (a.double() * b + c.double()).float()


def _f32(x: float) -> float:
    return torch.tensor(x, dtype=F32).item()


def _rel_terms(q32, rel, S, axis):
    """fp32 q . rel[qc - kc + S - 1] for every query and key coordinate kc: [n, T, S]."""
    T = S * S
    tab = q32 @ rel.float().t()                                   # [n, T, 2S - 1], fp32 sums over hd
    t = torch.arange(T)
    qc = t // S if axis == "h" else t % S
    idx = qc[:, None] - torch.arange(S)[None, :] + S - 1
    return tab.gather(2, idx.expand(tab.shape[0], T, S))


def _scale2(hd):
    return _f32(_f32(1.0 / _f32(math.sqrt(hd))) * _f32(LOG2E))


def _log2_logits(q, k, rel_h, rel_w, S, hd):
    """The flash / three-pass logits: fmaf(q.k, hd^-0.5 log2 e, rel_h log2 e + rel_w log2 e), all fp32."""
    T = S * S
    q32, k32 = q.float(), k.float()
    l2e = torch.tensor(LOG2E, dtype=F32)
    rh = _rel_terms(q32, rel_h, S, "h") * l2e
    rw = _rel_terms(q32, rel_w, S, "w") * l2e
    kk = torch.arange(T)
    return _fma(q32 @ k32.transpose(1, 2), _scale2(hd), rh[:, :, kk // S] + rw[:, :, kk % S])


def emulate_flash(qkv, rel_h, rel_w, n_seq, S, H, hd, p_dtype=torch.float16, no_alpha_tile=None):
    """attention.cu's wgmma kernel: online softmax over 64-key tiles, P and V in fp16 (p_dtype=bfloat16: P and V in
    bf16), l over the unrounded P, O / l rounded to bf16.  no_alpha_tile: that tile skips O's rescale."""
    T, BN = S * S, ea.BN
    nkt = (T + BN - 1) // BN
    q, k, v = _split(qkv, n_seq, S, H, hd)
    t = _log2_logits(q, k, rel_h, rel_w, S, hd)
    t = torch.cat([t, torch.full((*t.shape[:2], nkt * BN - T), -math.inf)], dim=2)
    vv = v.float().to(p_dtype).float()
    vv = torch.cat([vv, torch.zeros(vv.shape[0], nkt * BN - T, hd)], dim=1)
    m = torch.full((*t.shape[:2], 1), -math.inf)
    l = torch.zeros_like(m)
    o = torch.zeros(*t.shape[:2], hd)
    for j in range(nkt):
        tj = t[..., j * BN:(j + 1) * BN]
        m_new = torch.maximum(m, tj.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new)
        l = l * alpha
        if j != no_alpha_tile:
            o = o * alpha
        m = m_new
        p = torch.exp2(tj - m)
        l = l + p.sum(-1, keepdim=True)
        o = o + p.to(p_dtype).float() @ vv[:, j * BN:(j + 1) * BN]
    return _merge((o * (1.0 / l)).to(torch.bfloat16), n_seq, S, H, hd)


def emulate_simt(qkv, rel_h, rel_w, n_seq, S, H, hd, sum_one_key_fewer=False):
    """vit_attention_simt_kernel: one key at a time, fp32 throughout, expf, bf16 output.  sum_one_key_fewer: the row
    sum misses the last key."""
    T = S * S
    q, k, v = (x.float() for x in _split(qkv, n_seq, S, H, hd))
    scale = _f32(1.0 / _f32(math.sqrt(hd)))
    rh, rw = _rel_terms(q, rel_h, S, "h"), _rel_terms(q, rel_w, S, "w")
    m = torch.full((*q.shape[:2], 1), -math.inf)
    l = torch.zeros_like(m)
    o = torch.zeros_like(q)
    for key in range(T):
        s = (q @ k[:, key].unsqueeze(-1)) * scale + rh[:, :, key // S:key // S + 1] + rw[:, :, key % S:key % S + 1]
        mn = torch.maximum(m, s)
        a, pe = torch.exp(m - mn), torch.exp(s - mn)
        l = l * a + (0.0 if sum_one_key_fewer and key == T - 1 else pe)
        o = o * a + pe * v[:, key].unsqueeze(1)
        m = mn
    return _merge((o / l).to(torch.bfloat16), n_seq, S, H, hd)


def emulate_three_pass(qkv, rel_h, rel_w, n_seq, S, H, hd):
    """attention_generic.cu: fp32 scores and tables, base-2 softmax with ex2, P = bf16(p / l), bf16 P V over T."""
    q, k, v = _split(qkv, n_seq, S, H, hd)
    t = _log2_logits(q, k, rel_h, rel_w, S, hd)
    p = torch.exp2(t - t.amax(-1, keepdim=True))
    P = (p * (1.0 / p.sum(-1, keepdim=True))).to(torch.bfloat16)
    return _merge((P.float() @ v.float()).to(torch.bfloat16), n_seq, S, H, hd)


def emulate_softmax_bias(scores, tab, NT, S, scale):
    """attn_softmax_bias_kernel on rows 0 .. len(scores) of its input."""
    T = S * S
    q = torch.arange(scores.shape[0]) % T
    qh, qw = q // S, q % S
    kk = torch.arange(S)
    l2e = torch.tensor(LOG2E, dtype=F32)
    bh = tab.gather(1, qh[:, None] - kk[None, :] + S - 1) * l2e
    bw = tab.gather(1, NT + qw[:, None] - kk[None, :] + S - 1) * l2e
    key = torch.arange(T)
    t = _fma(scores[:, :T], _f32(_f32(scale) * _f32(LOG2E)), bh[:, key // S] + bw[:, key % S])
    p = torch.exp2(t - t.amax(-1, keepdim=True))
    return (p * (1.0 / p.sum(-1, keepdim=True))).to(torch.bfloat16)


def _ratio(out, ref, tol):
    return ea.max_ratio((out.double() - ref).abs(), tol)


# ---------------------------------------------------------------------------------------------------- pinning
def _hf_attention(qkv64, rel_h, rel_w, B, S, H, hd, window):
    """transformers' SamVisionAttention in float64 on the given qkv rows: its qkv Linear replaced by the identity
    (the input is the qkv tensor itself) and its proj by an identity Linear, so the output is the attention core."""
    from transformers.models.sam.modeling_sam import SamVisionAttention, SamVisionConfig
    D = H * hd
    cfg = SamVisionConfig(hidden_size=D, num_attention_heads=H, window_size=window, image_size=16 * S, patch_size=16)
    att = SamVisionAttention(cfg, window).double()
    assert att.rel_pos_h.shape == rel_h.shape
    with torch.no_grad():
        att.proj.weight.copy_(torch.eye(D, dtype=torch.float64))
        att.proj.bias.zero_()
        att.rel_pos_h.copy_(rel_h.double())
        att.rel_pos_w.copy_(rel_w.double())
    att.qkv = torch.nn.Identity()
    out, _ = att(qkv64.view(B, S, S, 3 * D))
    return out.reshape(B * S * S, D)


@pytest.mark.parametrize("S,window", [(14, 14), (32, 0)])
@pytest.mark.parametrize("hd", [64, 80])
def test_reference_matches_hf_float64(S, window, hd):
    B, H = 2, 2
    qkv, rh, rw = ea.inputs("tables15", B, S, H, hd, seed=S + hd)
    qkv64 = qkv.double()
    ref = ea.attention(qkv64, rh, rw, B, S, H, hd)
    hf = _hf_attention(qkv64, rh, rw, B, S, H, hd, window)
    err = (ref - hf).abs().max().item()
    assert err <= 2e-6 * ref.abs().max().item(), err
    # restate's fp32 core on the same operands (its softmax is fp32 too)
    q, k, v = (x.float() for x in _split(qkv, B, S, H, hd))
    core = _merge(restate.vit_attention_core(q, k, v, rh.float(), rw.float(), S), B, S, H, hd)
    err32 = (ref - core.double()).abs().max().item()
    assert err32 <= 2e-5 * ref.abs().max().item(), err32


def test_hf_pinning_sees_a_wrong_reference():
    """The HF comparison above is not vacuous: a reference with the rel-pos terms of the wrong axis fails it."""
    B, S, H, hd = 1, 14, 2, 64
    qkv, rh, rw = ea.inputs("tables15", B, S, H, hd, seed=3)
    hf = _hf_attention(qkv.double(), rh, rw, B, S, H, hd, 14)
    bad = ea.attention(qkv.double(), rw, rh, B, S, H, hd)
    assert (bad - hf).abs().max().item() > 1e-2


# ---------------------------------------------------------------------------------------------------- window maps
@pytest.mark.parametrize("grid", [14, 32, 48, 64, 80])
def test_window_maps_are_partition_and_unpartition(grid):
    from rsprompter_b200.sam_encoder import window_maps
    B, ws, C = 2, 14, 5
    wmap, n_win = window_maps(B, grid, ws, torch.device("cpu"))
    assert n_win == math.ceil(grid / ws) ** 2
    assert wmap.dtype == torch.int32 and wmap.numel() == B * n_win * ws * ws
    g = torch.Generator().manual_seed(grid)
    x = torch.randn(B, grid, grid, C, generator=g)
    # gather: row r of the windowed sequences is token wmap[r] (0 for padding), as LN1 reads it
    rows = x.reshape(-1, C)
    keep = wmap >= 0
    gathered = torch.zeros(wmap.numel(), C)
    gathered[keep] = rows[wmap[keep].long()]
    part, padded = restate.window_partition(x, ws)
    assert torch.equal(gathered.view(-1, ws, ws, C), part)
    # scatter: windowed row r goes to token wmap[r], padding rows are dropped, as the attention store writes them
    w = torch.randn(B * n_win, ws, ws, C, generator=g)
    out = torch.full((B * grid * grid, C), float("nan"))
    out[wmap[keep].long()] = w.reshape(-1, C)[keep]
    assert torch.equal(out.view(B, grid, grid, C), restate.window_unpartition(w, ws, padded, (grid, grid)))
    assert torch.equal(wmap[keep].sort().values, torch.arange(B * grid * grid, dtype=torch.int32))


# ---------------------------------------------------------------------------------------------------- bounds hold
@pytest.mark.parametrize("kind", ea.KINDS)
@pytest.mark.parametrize("S,hd", [(14, 80), (14, 64), (32, 80), (64, 64)])
def test_flash_emulation_within_bound(kind, S, hd):
    if S == 64 and kind not in ("random", "last_key", "rising", "fp16_edge"):
        pytest.skip("S = 64 on the CPU: the kinds whose edges depend on the 64 key tiles")
    qkv, rh, rw = ea.inputs(kind, **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    emu = emulate_flash(qkv, rh, rw, 1, S, 2, hd)
    assert torch.isfinite(emu.float()).all()
    r = _ratio(emu, ref, ea.flash_tol(qkv, rh, rw, 1, S, 2, hd, ref))
    print(f"flash emulation {kind} S={S} hd={hd}: max|err|/tol {r:.3f}")
    assert r <= 1.0
    if kind == "one_hot":
        assert torch.equal(emu, _split(qkv, 1, S, 2, hd)[2].reshape(2, S * S, hd).permute(1, 0, 2).reshape(-1, 2 * hd))


def test_flash_fp16_overflow_edge():
    """|v| = 65280 stays finite (it is fp16-representable); the next bf16 value, 65536, becomes inf in fp16."""
    qkv, rh, rw = ea.inputs("uniform", 1, 14, 1, 64)
    qkv[:, 128] = ea.FP16_V_MAX
    assert torch.isfinite(emulate_flash(qkv, rh, rw, 1, 14, 1, 64).float()).all()
    qkv[:, 128] = 65536.0
    assert not torch.isfinite(emulate_flash(qkv, rh, rw, 1, 14, 1, 64).float()).all()


@pytest.mark.parametrize("kind", ea.KINDS)
@pytest.mark.parametrize("S,hd", [(14, 80), (14, 64)])
def test_simt_emulation_within_bound(kind, S, hd):
    qkv, rh, rw = ea.inputs(kind, **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    emu = emulate_simt(qkv, rh, rw, 1, S, 2, hd)
    r = _ratio(emu, ref, ea.simt_tol(qkv, rh, rw, 1, S, 2, hd, ref))
    print(f"simt emulation {kind} S={S} hd={hd}: max|err|/tol {r:.3f}")
    assert r <= 1.0


@pytest.mark.parametrize("kind", ea.KINDS)
@pytest.mark.parametrize("hd", [64, 80])
def test_three_pass_emulation_within_bound(kind, hd):
    S = 48
    qkv, rh, rw = ea.inputs(kind, **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    emu = emulate_three_pass(qkv, rh, rw, 1, S, 2, hd)
    r = _ratio(emu, ref, ea.three_pass_tol(qkv, rh, rw, 1, S, 2, hd, ref))
    print(f"three-pass emulation {kind} hd={hd}: max|err|/tol {r:.3f}")
    assert r <= 1.0


def test_softmax_bias_emulation_within_bound():
    S, NT = 48, 112
    T = S * S
    scores, tab = ea.softmax_bias_inputs(S, T, NT, T + 4, 2 * NT + 8, seed=5)
    ref = ea.softmax_bias(scores, tab, NT, S, 0.125)
    emu = emulate_softmax_bias(scores, tab, NT, S, 0.125)
    r = _ratio(emu, ref, ea.softmax_bias_tol(scores, tab, NT, S, 0.125, ref))
    print(f"softmax_bias emulation: max|err|/tol {r:.3f}")
    assert r <= 1.0


# ---------------------------------------------------------------------------------------------------- bug distance
def _far(bug, ref, tol, what):
    r = _ratio(bug, ref, tol)
    print(f"{what}: {r:.1f} x the bound")
    assert r > FAR, f"{what}: the bug variant is only {r:.1f} x the tolerance away"


def _transpose_keys(qkv, n_seq, S, H, hd):
    """K and V rows of each sequence permuted by (kh, kw) -> (kw, kh): the same softmax as a kernel that reads the
    bias of key (kh, kw) at (kw, kh)."""
    D = H * hd
    x = qkv.reshape(n_seq, S, S, 3 * D).clone()
    x[..., D:] = x[..., D:].transpose(1, 2)
    return x.reshape(n_seq * S * S, 3 * D)


def _shift(rel):
    """Table row t + 1 read for row t (index q - k + S instead of q - k + S - 1), zero past the end (TMA's fill)."""
    return torch.cat([rel[1:], torch.zeros_like(rel[:1])])


def _with_padded_keys(qkv, rh, rw, n_seq, S, H, hd, n_pad):
    """The reference with n_pad extra keys of logit 0 and value 0 in every (sequence, head)."""
    T = S * S
    out = torch.empty(n_seq * T, H * hd, dtype=torch.float64)
    for seq, head, v, lg, _ in ea.blocks(qkv, rh, rw, n_seq, S, H, hd):
        lg = torch.cat([lg, torch.zeros(*lg.shape[:2], n_pad, dtype=lg.dtype)], dim=2)
        v = torch.cat([v, torch.zeros(v.shape[0], n_pad, hd, dtype=v.dtype)], dim=1)
        out.view(n_seq, T, H, hd)[seq, :, head] = torch.softmax(lg, -1) @ v
    return out


@pytest.mark.parametrize("S,hd", [(14, 64), (14, 80), (32, 64), (32, 80)])
def test_reference_bugs_are_far(S, hd):
    """Index and layout bugs of the rel-pos bias, restated on the reference, on the GPU test's random input."""
    n_seq, H = FEW["n_seq"], FEW["H"]
    qkv, rh, rw = ea.inputs("random", n_seq, S, H, hd)
    ref = ea.attention(qkv, rh, rw, n_seq, S, H, hd)
    tol = ea.flash_tol(qkv, rh, rw, n_seq, S, H, hd, ref)
    tab_qkv, trh, trw = ea.inputs("tables15", n_seq, S, H, hd)
    tref = ea.attention(tab_qkv, trh, trw, n_seq, S, H, hd)
    ttol = ea.flash_tol(tab_qkv, trh, trw, n_seq, S, H, hd, tref)
    for (x, a, b, r, t) in ((qkv, rh, rw, ref, tol), (tab_qkv, trh, trw, tref, ttol)):
        _far(ea.attention(x, b, a, n_seq, S, H, hd), r, t, "rel_h and rel_w swapped")
        _far(ea.attention(x, _shift(a), _shift(b), n_seq, S, H, hd), r, t, "table index q - k + S")
        _far(ea.attention(_transpose_keys(x, n_seq, S, H, hd), a, b, n_seq, S, H, hd), r, t, "kh and kw transposed")
        sc = hd ** -0.5
        _far(ea.attention(x, a.double() * sc, b.double() * sc, n_seq, S, H, hd), r, t, "scale on the rel-pos q")
    if S == 14:
        _far(_with_padded_keys(qkv, rh, rw, n_seq, S, H, hd, 64 * 4 - S * S), ref, tol, "keys 196-255 at logit 0")


@pytest.mark.parametrize("S,hd", [(14, 64), (14, 80), (32, 64), (32, 80), (64, 80)])
def test_dropped_rescale_is_far(S, hd):
    """One tile's O rescale dropped (the last one, where the running max rises again), on the rising input."""
    qkv, rh, rw = ea.inputs("rising", **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    tol = ea.flash_tol(qkv, rh, rw, 1, S, 2, hd, ref)
    nkt = (S * S + ea.BN - 1) // ea.BN
    _far(emulate_flash(qkv, rh, rw, 1, S, 2, hd, no_alpha_tile=nkt - 1), ref, tol, "alpha dropped in the last tile")


@pytest.mark.parametrize("S,hd", [(14, 64), (14, 80)])
def test_simt_short_row_sum_is_far(S, hd):
    """The SIMT kernel's row sum over one key fewer, on the input whose last key is every row's sharpest."""
    qkv, rh, rw = ea.inputs("last_key", **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    tol = ea.simt_tol(qkv, rh, rw, 1, S, 2, hd, ref)
    _far(emulate_simt(qkv, rh, rw, 1, S, 2, hd, sum_one_key_fewer=True), ref, tol, "SIMT row sum without key T-1")


@pytest.mark.parametrize("S,hd", [(14, 64), (14, 80), (32, 80), (64, 64)])
def test_bf16_p_is_outside_the_flash_bound(S, hd):
    """P in bf16 on the flash path.  No input can put it 10x outside the flash bound: the bound carries U11 sum_j w_j
    |v_j| for the fp16 rounding of P, and bf16 rounding of P costs at most U8 = 8 U11 of the same sum.  The p_tie
    input comes closest: every P sits just off a bf16 rounding tie, on the side that pushes each term P_j v_j the same
    way, while the output cancels to about 0 (so its own bf16 rounding adds nothing to the bound).  There the bug lands
    5.7-6.6x outside the bound for T <= 1024 and 3.6x at T = 4096, where the bound's fp32 accumulation terms (2T U24)
    reach the size of its fp16 term.  The GPU test runs the same input, so it would report the bug."""
    qkv, rh, rw = ea.inputs("p_tie", **FEW, S=S, hd=hd)
    ref = ea.attention(qkv, rh, rw, 1, S, 2, hd)
    tol = ea.flash_tol(qkv, rh, rw, 1, S, 2, hd, ref)
    r = _ratio(emulate_flash(qkv, rh, rw, 1, S, 2, hd, p_dtype=torch.bfloat16), ref, tol)
    print(f"P in bf16: {r:.1f} x the bound")
    assert r > (5.0 if S <= 32 else 3.0)
