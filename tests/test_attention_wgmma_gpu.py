"""The wgmma ViT attention kernel at the shapes the encoders run, against the fp32 SIMT restatement of the same
attention on the GPU: ViT-H and ViT-B windows (through the window un-partition scatter) and global grids, S = 32,
sharp logits where the online rescaling matters, a grid whose last wave of CTAs is partial, and repeatability."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(n_seq, S, H, hd, qk_scale, tab_scale, seed):
    g = torch.Generator().manual_seed(seed)
    T, D = S * S, H * hd
    qkv = (torch.randn(n_seq * T, 3 * D, generator=g) * qk_scale).to(torch.bfloat16).cuda()
    rh = (torch.randn(2 * S - 1, hd, generator=g) * tab_scale).to(torch.bfloat16).cuda()
    rw = (torch.randn(2 * S - 1, hd, generator=g) * tab_scale).to(torch.bfloat16).cuda()
    return qkv, rh, rw


def _rel_err(got, ref):
    return (got.float() - ref.float()).abs().max().item() / max(ref.float().abs().max().item(), 1e-6)


@pytest.mark.parametrize("n_seq,S,H,hd,qk_scale,tab_scale", [
    (8, 64, 16, 80, 1.0, 0.2),     # ViT-H global
    (2, 64, 12, 64, 1.0, 0.2),     # ViT-B global
    (3, 32, 16, 80, 1.0, 0.2),     # 512^2 input: S = 32
    (5, 32, 12, 64, 1.0, 0.2),
    (2, 64, 3, 64, 3.0, 1.5),      # sharp logits: the running max moves across key tiles
    (1, 64, 2, 80, 3.0, 1.5),
    (133, 14, 16, 80, 1.0, 0.2),   # 4256 CTAs: the last wave on 132 SMs is partial
    (50, 14, 12, 64, 3.0, 1.5),
])
def test_wgmma_attention_matches_simt(n_seq, S, H, hd, qk_scale, tab_scale):
    from rsprompter_b200 import _lib
    qkv, rh, rw = _inputs(n_seq, S, H, hd, qk_scale, tab_scale, seed=n_seq * 100 + S + hd)
    out = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd)
    ref = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd, simt=True)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert _rel_err(out, ref) < 1.5e-2


@pytest.mark.parametrize("batch,H,hd", [(8, 16, 80), (8, 12, 64)])
def test_wgmma_window_attention_scatter(batch, H, hd):
    """200 windows of a 64 x 64 grid, stored straight into the un-partitioned token rows (padding rows dropped)."""
    from rsprompter_b200 import _lib
    from rsprompter_b200.sam_encoder import window_maps
    S, grid = 14, 64
    rmap, nw = window_maps(batch, grid, S, torch.device("cuda"))
    n_seq = batch * nw
    qkv, rh, rw = _inputs(n_seq, S, H, hd, 1.0, 0.2, seed=batch + H + hd)
    out_rows = batch * grid * grid
    out = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd, out_row_map=rmap, out_rows=out_rows)
    ref_win = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd, simt=True)
    torch.cuda.synchronize()
    keep = rmap >= 0
    ref = torch.empty_like(out)
    ref[rmap[keep].long()] = ref_win[keep]
    assert int(keep.sum()) == out_rows
    assert _rel_err(out, ref) < 1.5e-2


@pytest.mark.parametrize("n_seq,S,H,hd", [(4, 64, 16, 80), (60, 14, 16, 80)])
def test_wgmma_attention_is_deterministic(n_seq, S, H, hd):
    from rsprompter_b200 import _lib
    qkv, rh, rw = _inputs(n_seq, S, H, hd, 1.0, 0.2, seed=7)
    a = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd)
    b = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
