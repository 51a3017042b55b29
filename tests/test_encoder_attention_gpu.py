"""The ViT encoder's attention kernels one by one against the float64 restatements of oracle/encoder_attention.py.

Each case asserts |kernel - reference| <= tol element by element, tol derived from the path's rounding points
(oracle/encoder_attention.py, the *_tol functions): fp32 logits (the tensor cores' sums truncate), ex2 / expf, the
flash kernel's fp16 P and V and its per-tile rescale, the three-pass path's normalised bf16 P, fp32 sums over T keys
and the bf16 output.  It prints the worst max|err|/tol of each case.  Where the answer is exact it is asserted bit for
bit: on the one_hot input every query attends to itself only, so the output row is that token's v.  The inputs are
the builders of oracle/encoder_attention.py (tests/test_encoder_attention_cpu.py shows that plausible bugs land far
outside these bounds on them); the references run in float64 on the GPU, chunked over (sequence, head)."""
import pytest
import torch

from oracle import encoder_attention as ea

pytestmark = pytest.mark.gpu

SMS = 132
# (n_seq, H) with many more 128-row query tiles than SMs, so every persistent CTA runs several tiles and the Q buffers
# and the K / V ring wrap: 768, 384 and 1536 tiles.  (hd 80, S 64) is the one instantiation with a single Q buffer.
MANY = {14: (64, 6), 32: (4, 12), 64: (6, 8)}


def _check(out, ref, tol, what):
    assert torch.isfinite(out.float()).all(), f"{what}: non-finite output"
    err = (out.to(torch.float64) - ref).abs()
    ratio = (err / tol).max().item()
    print(f"{what}: max|err| {err.max().item():.3e}  max|err|/tol {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: max |err| / tol = {ratio:.3f}, max |err| = {err.max().item():.3e}"


def _cuda(*ts):
    return [t.cuda() for t in ts]


def _v(qkv, H, hd):
    return qkv[:, 2 * H * hd:]


def _flash_case(kind, n_seq, S, H, hd, what):
    from rsprompter_b200 import _lib
    qkv, rh, rw = _cuda(*ea.inputs(kind, n_seq, S, H, hd))
    out = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd)
    torch.cuda.synchronize()
    if kind == "one_hot":
        assert torch.equal(out, _v(qkv, H, hd)), f"{what} {kind}: not the attended key's v"
    ref = ea.attention(qkv, rh, rw, n_seq, S, H, hd)
    _check(out, ref, ea.flash_tol(qkv, rh, rw, n_seq, S, H, hd, ref), f"{what} {kind}")


@pytest.mark.parametrize("tiles", ["few", "many"])
@pytest.mark.parametrize("S", [14, 32, 64])
@pytest.mark.parametrize("hd", [64, 80])
def test_flash_instantiation(hd, S, tiles):
    """All six instantiations of the wgmma kernel on every builder input: once with fewer query tiles than SMs
    (n_seq = 1, H = 2), once with several tiles per persistent CTA."""
    n_seq, H = (1, 2) if tiles == "few" else MANY[S]
    n_tiles = n_seq * H * ((S * S + 127) // 128)
    assert (n_tiles < SMS) if tiles == "few" else (n_tiles >= 2.5 * SMS)
    for kind in ea.KINDS:
        _flash_case(kind, n_seq, S, H, hd, f"flash hd={hd} S={S} n_seq={n_seq} H={H}")


@pytest.mark.parametrize("name,n_seq,S,H,hd", [
    ("ViT-H global", 8, 64, 16, 80),
    ("ViT-B global", 8, 64, 12, 64),
])
def test_flash_production_global(name, n_seq, S, H, hd):
    for kind in ("random", "sharp", "rising"):
        _flash_case(kind, n_seq, S, H, hd, name)


@pytest.mark.parametrize("name,H,hd", [("ViT-H windows", 16, 80), ("ViT-B windows", 12, 64)])
def test_flash_production_windows(name, H, hd):
    """200 windows (batch 8 of a 64 x 64 grid) with the encoder's padding rows (the qkv bias vector)."""
    from rsprompter_b200 import _lib
    qkv, rh, rw, _, n_win = ea.window_inputs(8, 64, H, hd)
    qkv, rh, rw = _cuda(qkv, rh, rw)
    n_seq = 8 * n_win
    assert n_seq == 200
    out = _lib.vit_attention(qkv, rh, rw, n_seq, 14, H, hd)
    torch.cuda.synchronize()
    ref = ea.attention(qkv, rh, rw, n_seq, 14, H, hd)
    _check(out, ref, ea.flash_tol(qkv, rh, rw, n_seq, 14, H, hd, ref), name)


@pytest.mark.parametrize("grid", [32, 48, 64, 80])
@pytest.mark.parametrize("H,hd", [(3, 80), (2, 64)])
def test_scatter_store(grid, H, hd):
    """rsp_vit_attention with out_row_map: windows of a B = 2 grid (padded to 42 / 56 / 70 / 84) stored through window_maps
    into a NaN-prefilled [B g g, D] output.  Every token row is written and within the bound; with a second map that
    drops some real rows (-1), exactly those rows keep the NaN."""
    from rsprompter_b200 import _lib
    B = 2
    qkv, rh, rw, wmap, n_win = ea.window_inputs(B, grid, H, hd)
    qkv, rh, rw, wmap = _cuda(qkv, rh, rw, wmap)
    n_seq, rows, Dm = B * n_win, B * grid * grid, H * hd
    ref_w = ea.attention(qkv, rh, rw, n_seq, 14, H, hd)
    tol_w = ea.flash_tol(qkv, rh, rw, n_seq, 14, H, hd, ref_w)
    keep = wmap >= 0
    ref = torch.full((rows, Dm), float("nan"), dtype=torch.float64, device="cuda")
    tol = torch.full_like(ref, float("nan"))
    ref[wmap[keep].long()] = ref_w[keep]
    tol[wmap[keep].long()] = tol_w[keep]
    assert not ref.isnan().any()

    out = torch.full((rows, Dm), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.vit_attention(qkv, rh, rw, n_seq, 14, H, hd, out=out, out_row_map=wmap, out_rows=rows)
    torch.cuda.synchronize()
    assert not out.isnan().any()
    _check(out, ref, tol, f"scatter grid={grid} H={H} hd={hd}")

    r = torch.arange(wmap.numel(), device="cuda")
    drop = keep & (r % 7 == 3)
    m2 = torch.where(drop, torch.full_like(wmap, -1), wmap)
    gone = torch.zeros(rows, dtype=torch.bool, device="cuda")
    gone[wmap[drop].long()] = True
    out2 = torch.full((rows, Dm), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.vit_attention(qkv, rh, rw, n_seq, 14, H, hd, out=out2, out_row_map=m2, out_rows=rows)
    torch.cuda.synchronize()
    assert gone.any() and out2[gone].isnan().all()
    assert not out2[~gone].isnan().any()
    assert torch.equal(out2[~gone], out[~gone])


@pytest.mark.parametrize("S", [14, 32, 64])
@pytest.mark.parametrize("hd", [64, 80])
def test_simt(S, hd):
    """rsp_vit_attention_simt (the reference of test_attention_wgmma_gpu.py) against float64 with its own bound."""
    from rsprompter_b200 import _lib
    n_seq, H = 2, 2
    for kind in ea.KINDS:
        qkv, rh, rw = _cuda(*ea.inputs(kind, n_seq, S, H, hd))
        out = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd, simt=True)
        torch.cuda.synchronize()
        if kind == "one_hot":
            assert torch.equal(out, _v(qkv, H, hd))
        ref = ea.attention(qkv, rh, rw, n_seq, S, H, hd)
        _check(out, ref, ea.simt_tol(qkv, rh, rw, n_seq, S, H, hd, ref), f"simt hd={hd} S={S} {kind}")


@pytest.mark.parametrize("n_seq", [1, 2])
@pytest.mark.parametrize("S", [48, 80])
@pytest.mark.parametrize("hd", [64, 80])
def test_three_pass(S, hd, n_seq):
    """vit_attention on the grids the flash kernel does not specialise (768^2 / 1280^2 inputs): split_heads,
    transpose_cols, the grouped Q K^T, the table GEMM, attn_softmax_bias and the grouped P V."""
    from rsprompter_b200 import _lib
    H = 2
    for kind in ea.KINDS:
        qkv, rh, rw = _cuda(*ea.inputs(kind, n_seq, S, H, hd))
        out = _lib.vit_attention(qkv, rh, rw, n_seq, S, H, hd)
        torch.cuda.synchronize()
        if kind == "one_hot":
            assert torch.equal(out, _v(qkv, H, hd))
        ref = ea.attention(qkv, rh, rw, n_seq, S, H, hd)
        _check(out, ref, ea.three_pass_tol(qkv, rh, rw, n_seq, S, H, hd, ref),
               f"three-pass hd={hd} S={S} n_seq={n_seq} {kind}")


@pytest.mark.parametrize("S,groups,pad", [
    (48, 2, True),     # NV = 3 (T <= 3072); two row groups in one launch; every leading dimension padded
    (48, 1, False),
    (80, 1, True),     # NV = 7 (T <= 7168)
    (128, 1, True),    # NV = 16 (T <= 16384)
])
def test_attn_softmax_bias(S, groups, pad):
    """rsp_attn_softmax_bias alone against a float64 softmax of the same fp32 scores and tables.  pad: lds / ldt / ldp
    larger than needed and NT 16 rows past the padded 2S - 1; the columns the kernel must not read are NaN, the
    columns of P it must not write are NaN-prefilled."""
    from rsprompter_b200 import _lib
    T = S * S
    n_rows = groups * T
    NT = (2 * S - 1 + 15) // 16 * 16 + (16 if pad else 0)
    lds, ldt, ldp = (T + 36, 2 * NT + 8, T + 12) if pad else (T, 2 * NT, T)
    scores, tab = _cuda(*ea.softmax_bias_inputs(S, n_rows, NT, lds, ldt, seed=S + groups))
    P = torch.full((n_rows, ldp), float("nan"), dtype=torch.bfloat16, device="cuda")
    scale = 80 ** -0.5
    st = _lib._lib.rsp_attn_softmax_bias(scores.data_ptr(), lds, tab.data_ptr(), ldt, NT, P.data_ptr(), ldp, n_rows,
                                          T, S, scale, _lib._stream())
    torch.cuda.synchronize()
    assert st == 0
    assert P[:, T:].isnan().all()
    worst, worst_err = 0.0, 0.0
    step = 1024
    for r0 in range(0, n_rows, step):
        sl = slice(r0, min(n_rows, r0 + step))
        ref = ea.softmax_bias(scores[sl], tab[sl], NT, S, scale, row0=r0)
        tol = ea.softmax_bias_tol(scores[sl], tab[sl], NT, S, scale, ref, row0=r0)
        err = (P[sl, :T].double() - ref).abs()
        worst, worst_err = max(worst, (err / tol).max().item()), max(worst_err, err.max().item())
    print(f"attn_softmax_bias S={S} groups={groups} pad={pad}: max|err| {worst_err:.3e}  max|err|/tol {worst:.3f}")
    assert worst <= 1.0


def _guarded(numel):
    """A NaN-prefilled bf16 buffer with 256 guard elements past numel."""
    buf = torch.full((numel + 256,), float("nan"), dtype=torch.bfloat16, device="cuda")
    return buf, buf[:numel]


@pytest.mark.parametrize("T", [100, 196, 2304])
def test_split_heads_and_transpose_cols(T):
    """Exact copies: column offsets, ld > 3D, T and C not multiples of the 32 x 32 transpose tile; nothing is
    written past the output."""
    from rsprompter_b200 import _lib
    n_seq, H, hd = 2, 3, 80
    Dm = H * hd
    ld = 3 * Dm + 24
    g = torch.Generator().manual_seed(T)
    x = torch.randn(n_seq * T, ld, generator=g).to(torch.bfloat16).cuda()
    x3 = x.view(n_seq, T, ld)
    for col0 in (0, 8, Dm, 2 * Dm + 16):
        buf, out = _guarded(n_seq * H * T * hd)
        st = _lib._lib.rsp_split_heads(x.data_ptr(), ld, col0, H, hd, n_seq, T, out.data_ptr(), _lib._stream())
        torch.cuda.synchronize()
        assert st == 0
        want = x3[:, :, col0:col0 + Dm].reshape(n_seq, T, H, hd).permute(0, 2, 1, 3).contiguous()
        assert torch.equal(out.view(n_seq, H, T, hd), want), col0
        assert buf[out.numel():].isnan().all()
    for col0, C in ((2 * Dm, Dm), (3, 77), (Dm + 5, 40), (ld - 33, 33)):
        buf, out = _guarded(n_seq * C * T)
        st = _lib._lib.rsp_transpose_cols(x.data_ptr(), ld, col0, C, n_seq, T, out.data_ptr(), _lib._stream())
        torch.cuda.synchronize()
        assert st == 0
        assert torch.equal(out.view(n_seq, C, T), x3[:, :, col0:col0 + C].transpose(1, 2)), (col0, C)
        assert buf[out.numel():].isnan().all()
