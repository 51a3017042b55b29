"""The float64 references of the query head's kernels (oracle/query_kernels.py), checked without a GPU:
  * pinned to the restatements they stand in for: ms_deform_core to restate_query.ms_deform_attn with identity value
    and output projections, grouped_gemm to one matrix product per group, sam_mask_embed_src to
    restate.sam_mask_embedding and the per-prompt image embedding of restate_query.forward_head;
  * bug distance: on the inputs of tests/test_query_kernels_gpu.py, a plausible kernel defect, restated on the
    reference, lands more than 10x the tolerance away from the right answer, so the GPU test would fail on it."""
import pytest
import torch
import torch.nn.functional as F

from oracle import decoder_kernels as dk
from oracle import query_kernels as qk
from oracle import restate, restate_query

FAR = 10.0
SHAPES = [(6, 10), (12, 20), (3, 5), (1, 1)]


def _far(bug, ref, tol, what):
    ok = ~ref.isnan()
    r = dk.max_ratio((bug - ref).abs()[ok], tol[ok])
    assert r > FAR, f"{what}: the defect is only {r:.1f} x the tolerance away"


# ---------------------------------------------------------------------------------------------------- MSDeformAttn
def test_ms_deform_core_matches_restate():
    """ms_deform_core on offsets / logits computed from the query is restate_query.ms_deform_attn with identity value
    and output projections (its output minus the identity)."""
    shapes, P, B, E = SHAPES[:3], 4, 2, 128
    L, NQ = len(shapes), sum(h * w for h, w in shapes)
    g = torch.Generator().manual_seed(0)
    q = torch.randn(B, NQ, E, generator=g)
    sd = {"value_proj.weight": torch.eye(E), "value_proj.bias": torch.zeros(E),
          "output_proj.weight": torch.eye(E), "output_proj.bias": torch.zeros(E),
          "sampling_offsets.weight": 0.3 * torch.randn(8 * L * P * 2, E, generator=g),
          "sampling_offsets.bias": 2 * torch.randn(8 * L * P * 2, generator=g),
          "attention_weights.weight": 0.2 * torch.randn(8 * L * P, E, generator=g),
          "attention_weights.bias": torch.randn(8 * L * P, generator=g)}
    ref_pts = qk.deform_ref_points(shapes).float()[None, :, None].repeat(B, 1, L, 1)
    exp = restate_query.ms_deform_attn(sd, "", q, torch.zeros_like(q), ref_pts, shapes, 8, P) - q
    ow = torch.cat([F.linear(q.double(), sd["sampling_offsets.weight"].double(), sd["sampling_offsets.bias"].double()),
                    F.linear(q.double(), sd["attention_weights.weight"].double(),
                             sd["attention_weights.bias"].double())], dim=-1).reshape(B * NQ, -1)
    got = qk.ms_deform_core(q, ow, shapes, P)
    err = (got - exp.reshape(B * NQ, E).double()).abs().max().item()
    assert err < 1e-4, err


@pytest.mark.parametrize("hd", [16, 32])
@pytest.mark.parametrize("logits", ["normal", "spread", "equal"])
def test_ms_deform_defects_are_far(hd, logits):
    """A swapped (H, W) normaliser, reference points placed on the next level's grid, and level starts one pixel off
    all land far outside the tolerance."""
    P = 4
    value, ow = qk.deform_inputs(SHAPES, P, hd, 2, seed=hd, logits=logits)
    ref = qk.ms_deform_core(value, ow, SHAPES, P)
    tol = qk.ms_deform_tol(value, ow, SHAPES, P, ref)
    _far(qk.ms_deform_core(value, ow, SHAPES, P, norm=[(h, w) for h, w in SHAPES]), ref, tol, "H / W swapped")
    L = len(SHAPES)
    _far(qk.ms_deform_core(value, ow, SHAPES, P, ref=qk.deform_ref_points(SHAPES, level_of=lambda l: (l + 1) % L)),
         ref, tol, "reference point of another level")
    starts = [s + (1 if l else 0) for l, s in enumerate(qk.level_starts(SHAPES))]
    _far(qk.ms_deform_core(value, ow, SHAPES, P, starts=starts), ref, tol, "level start off by one")


def test_deform_inputs_reach_every_edge():
    """The offsets put samples exactly on pixel -1 and W of every level, outside it, and on half-integer positions."""
    P = 5
    value, ow = qk.deform_inputs(SHAPES, P, 16, 2, seed=3)
    B, NQ, L = 2, value.shape[1], len(SHAPES)
    off, _ = qk._deform_split(ow, B, NQ, L, P)
    wh = torch.tensor([[w, h] for h, w in SHAPES], dtype=torch.float64)
    pix = qk.deform_ref_points(SHAPES)[None, :, None, None, None, :] * wh[None, None, None, :, None, :] - 0.5 + off
    for l in range(L):
        x = pix[:, :, :, l, ..., 0]
        assert (x == -1).any() and (x == wh[l, 0]).any() and (x < -2).any() and (x > wh[l, 0] + 1).any()
        assert ((x * 2 == torch.round(x * 2)) & (x != torch.round(x))).any()


# ---------------------------------------------------------------------------------------------------- grouped GEMM
def test_grouped_gemm_matches_per_group_products():
    me, mf, back = qk.grouped_inputs(3, 100, 144, seed=1, C=64)
    ref = qk.grouped_gemm(me, mf, 144, 128, 144, back, out_rows=305)
    for b in range(3):
        exp = me[b * 128:b * 128 + 100].double() @ mf[b * 144:(b + 1) * 144].double().t()
        assert torch.equal(ref[b * 100:(b + 1) * 100], exp)
    assert ref[300:].isnan().all()


@pytest.mark.parametrize("hw_l", [144, 400, 1600])
def test_grouped_gemm_tail_defect_is_far(hw_l):
    """The last, partial 128-column tile reading group g + 1's weight rows (the rows right after group g's N) is far
    outside the tolerance: neighbouring images' features differ by a factor 10 or more (0 past the last group)."""
    B, N = 8, hw_l
    me, mf, back = qk.grouped_inputs(B, 100, hw_l, seed=hw_l, C=64)
    ref = qk.grouped_gemm(me, mf, N, 128, hw_l, back)
    tol = qk.grouped_gemm_tol(me, mf, N, 128, hw_l, ref, back, out_bf16=False)
    tail0 = N // 128 * 128
    bug = qk.grouped_gemm(me, mf, N, 128, hw_l, back,
                          w_of_col=lambda g, n: torch.where(n >= tail0, (g + 1) * hw_l + n, g * hw_l + n))
    _far(bug[:, tail0:], ref[:, tail0:], tol[:, tail0:], "tail columns from the next group")


# ---------------------------------------------------------------------------------------------------- mask embedding
def _mask_embedding_variant(weights, mpp, approximate="none", ln_dim=1, eps=1e-6):
    """SamMaskEmbedding in float64 with its GELU or its LayerNorm axis replaced (ln_dim 1: channels, as HF)."""
    w1, b1, g1, be1, w2, b2, g2, be2, w3, b3 = [t.double() for t in weights]

    def ln(x, g, b):
        u = x.mean(ln_dim, keepdim=True)
        s = (x - u).pow(2).mean(ln_dim, keepdim=True)
        return g.view(1, -1, 1, 1) * (x - u) / torch.sqrt(s + eps) + b.view(1, -1, 1, 1)

    h = F.gelu(ln(F.conv2d(mpp.double().unsqueeze(1), w1, b1, stride=2), g1, be1), approximate=approximate)
    h = F.gelu(ln(F.conv2d(h, w2, b2, stride=2), g2, be2), approximate=approximate)
    return qk._rows(F.conv2d(h, w3.reshape(256, 16, 1, 1), b3))


def test_mask_embed_src_matches_restate():
    """The source rows are restate.sam_mask_embedding plus the prompt's image embedding, as restate_query.forward_head
    pairs them (repeat_interleave of the images over their n_per_img prompts); src_pe adds the key PE."""
    N, hw, npi = 6, (8, 4), 3
    weights = qk.mask_embed_weights(seed=1)
    mpp, emb, pos = qk.mask_embed_inputs(N, hw, npi, seed=2)
    src, src_pe = qk.sam_mask_embed_src(mpp, weights, emb, pos, npi, hw)
    sd32 = {k: v.float() for k, v in qk.mask_embed_sd(weights).items()}
    dense = restate.sam_mask_embedding(sd32, mpp.unsqueeze(1))                      # fp32, as the restatement runs
    emb_img = emb.view(N // npi, *hw, 256).permute(0, 3, 1, 2)
    exp = (dense + torch.repeat_interleave(emb_img, npi, dim=0)).permute(0, 2, 3, 1).reshape(-1, 256)
    assert (src - exp.double()).abs().max().item() < 1e-4 * max(1.0, exp.abs().max().item())
    assert torch.equal(src_pe, src + pos.double().repeat(N, 1))
    assert torch.allclose(_mask_embedding_variant(weights, mpp), src - emb.double()[torch.arange(N) // npi].reshape(-1, 256),
                          rtol=0, atol=1e-12)


@pytest.mark.parametrize("mma", [False, True])
def test_mask_embed_defects_are_far(mma):
    """tanh GELU and a LayerNorm over the width instead of the channels land far outside both kernels' bounds."""
    N, hw, npi = 15, (16, 16), 5
    weights = qk.mask_embed_weights(seed=3)
    mpp, emb, pos = qk.mask_embed_inputs(N, hw, npi, seed=4)
    src, _ = qk.sam_mask_embed_src(mpp, weights, emb, pos, npi, hw)
    tol = qk.mask_embed_src_tol(mpp, weights, src, mma=mma)
    e = emb.double()[torch.arange(N) // npi].reshape(-1, 256)
    _far(_mask_embedding_variant(weights, mpp, approximate="tanh") + e, src, tol, "tanh GELU")
    _far(_mask_embedding_variant(weights, mpp, ln_dim=3) + e, src, tol, "LayerNorm over the wrong axis")
