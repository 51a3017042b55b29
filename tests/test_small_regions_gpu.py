"""SAM's small-region removal on the GPU: rsp_mask_small_regions_bits against oracle.restate_small_regions'
remove_small_regions over cv2, bit for bit with its changed flags and boxes, per mode; its repeatability; then
generate_masks(min_mask_region_area=A) against the oracle composition on structured decoder outputs, with the
argument's neutral value, batching, RLE strings, host synchronisations and the CLI."""
import json
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

MODES = ("holes", "islands")


def _contents(H, W, seed):
    """Masks bool [n, H, W]: empty, full, blobs, salt-and-pepper noise at several densities (0.45-0.6 sit near the
    8-connected percolation point), a checkerboard, diagonal lines, a serpentine and concentric rings."""
    rng = np.random.default_rng(seed)
    ys, xs = np.indices((H, W))
    g = torch.Generator().manual_seed(seed)
    field = F.interpolate(torch.randn(1, 1, max(2, H // 24), max(2, W // 24), generator=g), (H, W), mode="bilinear",
                          align_corners=False)[0, 0].numpy()
    # one path: full rows 0, 4, 8, ... joined at alternate ends
    serp = (ys % 4 == 0) | (xs == np.where((ys // 4) % 2 == 0, W - 1, 0))
    dist = np.sqrt((ys - H / 2) ** 2 + (xs - W / 2) ** 2)
    masks = [np.zeros((H, W), bool), np.ones((H, W), bool), field > 0.3]
    masks += [rng.random((H, W)) < d for d in (0.2, 0.45, 0.55, 0.6, 0.8)]
    masks += [(ys + xs) % 2 == 0, (xs - ys) % 7 == 0, serp, (dist // 3).astype(int) % 2 == 0]
    return np.stack(masks)


def _pack(masks, garbage_seed=None):
    """bool [n, H, W] -> the generator's bit rows uint8 [n, H, ceil(W / 16) * 2] on the GPU; garbage_seed: random
    bits in the padding past W."""
    n, H, W = masks.shape
    ld = (W + 15) // 16 * 2
    full = np.zeros((n, H, ld * 8), bool)
    full[..., :W] = masks
    if garbage_seed is not None:
        full[..., W:] = np.random.default_rng(garbage_seed).random((n, H, ld * 8 - W)) < 0.5
    return torch.from_numpy(np.packbits(full, axis=-1, bitorder="little")).cuda()


def _unpack(bits):
    return np.unpackbits(bits.cpu().numpy(), axis=-1, bitorder="little").astype(bool)


def _component_areas(masks, mode):
    import cv2
    out = []
    for m in masks:
        work = (~m if mode == "holes" else m).astype(np.uint8)
        out.append(cv2.connectedComponentsWithStats(work, 8)[2][1:, -1])
    return np.concatenate(out)


def _check_kernel(masks, area, mode, seed):
    from oracle.restate_small_regions import mask_to_box, remove_small_regions
    from rsprompter_b200 import _lib
    n, H, W = masks.shape
    out, changed, boxes = _lib.mask_small_regions_bits(_pack(masks, garbage_seed=seed), W, area, mode)
    clean = _lib.mask_small_regions_bits(_pack(masks), W, area, mode)
    assert torch.equal(out, clean[0]) and torch.equal(changed, clean[1]) and torch.equal(boxes, clean[2])
    got = _unpack(out)
    assert not got[..., W:].any()
    refs = []
    for i in range(n):
        ref, ch = remove_small_regions(masks[i], area, mode)
        assert (got[i, :, :W] == ref).all(), (mode, area, i)
        assert bool(changed[i]) == ch, (mode, area, i)
        refs.append(torch.from_numpy(np.asarray(ref, dtype=bool)))
    assert torch.equal(boxes.cpu().long(), mask_to_box(torch.stack(refs)))
    return changed.cpu()


@pytest.mark.parametrize("hw", [(1, 1), (1, 777), (555, 1), (2, 3), (333, 517), (601, 799), (1024, 1024)])
@pytest.mark.parametrize("mode", MODES)
def test_kernel_matches_cv2(hw, mode):
    """Every content at fixed thresholds and at a component's exact area A (not small) and A + 1 (small)."""
    H, W = hw
    masks = _contents(H, W, seed=H + W)
    areas = _component_areas(masks, mode)
    s = int(np.median(areas)) if len(areas) else 1
    changed = [_check_kernel(masks, a, mode, seed=a) for a in (2, 9, s, s + 1)]
    if H * W > 100:
        assert any(c.any() for c in changed) and any((~c).any() for c in changed)


@pytest.mark.parametrize("mode", MODES)
def test_kernel_matches_cv2_on_a_large_mask(mode):
    H, W = 3000, 4000
    masks = _contents(H, W, seed=5)[[2, 5, 10]]         # blobs, noise at 0.55, the serpentine
    for a in (3, 40):
        _check_kernel(masks, a, mode, seed=a)


# -------------------------------------------------------------------------------------------------- repeatability
def test_two_launches_give_identical_bytes_and_a_batch_equals_each_mask_alone():
    from rsprompter_b200 import _lib
    masks = _contents(1024, 1024, seed=11)
    bits = _pack(masks)
    W = masks.shape[2]
    for mode in MODES:
        a = _lib.mask_small_regions_bits(bits, W, 50, mode)
        b = _lib.mask_small_regions_bits(bits, W, 50, mode)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        for i in range(masks.shape[0]):
            one = _lib.mask_small_regions_bits(bits[i:i + 1].contiguous(), W, 50, mode)
            assert torch.equal(one[0][0], a[0][i]) and torch.equal(one[1][0], a[1][i]) and torch.equal(one[2][0], a[2][i])


# -------------------------------------------------------------------------------------------------- generate_masks
@pytest.fixture(scope="module")
def sam():
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch
    arch, darch = VISION_ARCHS["base"], SamDecoderArch()
    sd = {"shared_image_embedding.positional_embedding":
          synthetic.positional_embedding_state_dict(arch, 54)["positional_embedding"]}
    sd.update({"vision_encoder." + k: v for k, v in synthetic.vision_encoder_state_dict(arch, seed=51).items()})
    sd.update({"mask_decoder." + k: v for k, v in synthetic.mask_decoder_state_dict(darch, seed=52).items()})
    sd.update({"prompt_encoder." + k: v for k, v in synthetic.prompt_encoder_state_dict(darch, seed=53).items()})
    model = MODELS.build(dict(type="RSSamModel", hf_pretrain_name="facebook/sam-vit-base"))
    model.sam_model.load_state_dict(sd, strict=True)
    return dict(model=model.cuda().eval(), sd=sd)


def _image(hw, seed):
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, 8, 8, generator=g) * 255, hw, mode="bilinear", align_corners=False)[0]
    return (base + 20 * torch.rand(3, *hw, generator=g)).clamp(0, 255).to(torch.uint8)


def _spotty(n, seed):
    """Low-res logits of one localised blob per mask, with up to 4 small islands anywhere and up to 3 small holes in
    the blob: components on both sides of the areas used below, and boxes that shrink when islands go."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(256.), torch.arange(256.), indexing="ij")
    out = torch.empty(n, 256, 256)
    for i in range(n):
        c = 40 + 176 * torch.rand(2, generator=g)
        r = 15 + 35 * torch.rand(1, generator=g)
        low = (r * r - (ys - c[0]) ** 2 - (xs - c[1]) ** 2) / r
        for _ in range(int(torch.randint(0, 5, (1,), generator=g))):
            p, s = 256 * torch.rand(2, generator=g), 1.5 + 3 * torch.rand(1, generator=g)
            low = torch.maximum(low, (s * s - (ys - p[0]) ** 2 - (xs - p[1]) ** 2) / s)
        for _ in range(int(torch.randint(0, 4, (1,), generator=g))):
            p, s = c + 0.7 * r * (2 * torch.rand(2, generator=g) - 1), 1.5 + 3 * torch.rand(1, generator=g)
            low = torch.minimum(low, -(s * s - (ys - p[0]) ** 2 - (xs - p[1]) ** 2) / s)
        out[i] = low + 1e-3 * torch.randn(256, 256, generator=g)
    return out


def _between(values, q):
    v = torch.unique(values[torch.isfinite(values)].double())
    i = max(1, min(len(v) - 1, int(q * len(v))))
    return float((v[i - 1] + v[i]) / 2)


def _pairwise_iou(b):
    b = b.double()
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = torch.maximum(b[:, None, :2], b[None, :, :2])
    rb = torch.minimum(b[:, None, 2:], b[None, :, 2:])
    inter = (rb - lt).clamp(min=0).prod(-1)
    iou = inter / (area[:, None] + area[None, :] - inter)
    return iou[torch.triu(torch.ones_like(iou, dtype=torch.bool), 1)]


N_SIDE, N_PTS = 8, 64
CASES = {"u8_600x800": ((600, 800), (768, 1024)), "pixel_values": ((333, 517), (660, 1024))}
KEYS = ("masks", "scores", "stability_scores", "boxes", "points", "candidates")


def _inputs(case):
    if case == "u8_600x800":
        return dict(images=_image((600, 800), 2))
    g = torch.Generator().manual_seed(3)
    pv = torch.zeros(1, 3, 1024, 1024)
    pv[..., :660, :] = F.interpolate(torch.randn(1, 3, 16, 16, generator=g), (660, 1024), mode="bilinear",
                                     align_corners=False)
    return dict(pixel_values=pv, original_sizes=[(333, 517)], reshaped_input_sizes=[(660, 1024)])


class _Decoder:
    """Serves seeded structured outputs in place of the mask decoder, prompt by prompt from the device."""

    def __init__(self, low, iou):
        self.low, self.iou, self.served = low.cuda(), iou.cuda(), 0

    def __call__(self, emb_rows, pos_rows, sparse, hw, **kw):
        q0 = self.served
        self.served += sparse.shape[0]
        return self.low[q0:self.served], self.iou[q0:self.served]


def _structured(seed):
    low = _spotty(N_PTS * 3, seed).view(N_PTS, 3, 256, 256).contiguous()
    iou = torch.rand(N_PTS, 3, generator=torch.Generator().manual_seed(seed + 7))
    return low, iou


def _gen(sam, inputs, **kw):
    from rsprompter_b200 import mask_generation as mg
    return mg.generate_masks(sam["model"], **inputs, **kw)


def _thresholds(low, iou, hw, rs):
    from oracle import restate_mask_generation as R
    st = R.mask_stats(R.upscale(low, hw, rs).flatten(0, 1), 0.0, 1.0)
    pred = _between(iou.flatten(), 0.25)
    nms = _between(_pairwise_iou(st["boxes"][iou.flatten() > pred]), 0.7)
    return dict(pred_iou_thresh=pred, stability_score_thresh=0.0, crops_nms_thresh=nms)


GRID = dict(points_per_side=N_SIDE, points_per_batch=16)


def _same(a, b) -> bool:
    """Equal bytes (NaN stability scores of empty masks included)."""
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


@pytest.mark.parametrize("case", list(CASES))
def test_generate_masks_matches_oracle_composition(sam, case, monkeypatch):
    from oracle import restate_small_regions as S
    from rsprompter_b200 import mask_generation as mg
    (H, W), rs = CASES[case]
    low, iou = _structured(len(case))
    kw = _thresholds(low, iou, (H, W), rs)
    area = 150.5
    ref = S.generate(low, iou, (H, W), rs, min_mask_region_area=area, **kw)
    dec = _Decoder(low, iou)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    base = _gen(sam, _inputs(case), **GRID, **kw)[0]
    dec.served = 0
    got = _gen(sam, _inputs(case), min_mask_region_area=area, **GRID, **kw)[0]
    # the reference of the step itself: SAM's postprocess_small_regions on the masks the first stage kept
    pp = S.postprocess_small_regions(mg.masks_to_bool(base).cpu(), area, kw["crops_nms_thresh"])
    rows = pp["index"]
    k = base["masks"].shape[0]
    assert 0 < int(pp["changed"].sum()) < k                      # some masks change and some do not
    assert 0 < len(rows) < k                                     # the second NMS drops a mask the first kept
    assert not torch.equal(rows, torch.sort(rows).values)        # and the order changes
    assert torch.equal(got["candidates"], base["candidates"][rows])
    assert torch.equal(got["candidates"], ref["index"])
    for key in ("scores", "stability_scores", "points"):
        assert _same(got[key], base[key][rows.cuda()]), key
    assert torch.equal(mg.masks_to_bool(got).cpu(), pp["masks"])
    assert torch.equal(got["boxes"].cpu(), pp["boxes"]) and got["boxes"].dtype == torch.int64
    assert torch.equal(got["boxes"].cpu(), ref["boxes"])
    assert not _unpack(got["masks"])[..., W:].any()


@pytest.mark.parametrize("area", [1e19, 1e300])
def test_huge_area_makes_every_component_small(sam, area, monkeypatch):
    """A finite A beyond any 64-bit integer still means "every component is small": holes all filled, the largest
    island alone kept, every mask changed (as SAM's Python comparisons do)."""
    from oracle import restate_small_regions as S
    from rsprompter_b200 import mask_generation as mg
    case = "u8_600x800"
    (H, W), rs = CASES[case]
    low, iou = _structured(3)
    kw = _thresholds(low, iou, (H, W), rs)
    dec = _Decoder(low, iou)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    base = _gen(sam, _inputs(case), **GRID, **kw)[0]
    dec.served = 0
    got = _gen(sam, _inputs(case), min_mask_region_area=area, **GRID, **kw)[0]
    pp = S.postprocess_small_regions(mg.masks_to_bool(base).cpu(), area, kw["crops_nms_thresh"])
    assert pp["changed"].all() and len(pp["index"]) > 0
    assert torch.equal(got["candidates"], base["candidates"][pp["index"]])
    assert torch.equal(mg.masks_to_bool(got).cpu(), pp["masks"])
    assert torch.equal(got["boxes"].cpu(), pp["boxes"])


def test_workspace_budget_does_not_change_the_result(sam, monkeypatch):
    from rsprompter_b200 import mask_generation as mg
    case = "pixel_values"
    (H, W), rs = CASES[case]
    low, iou = _structured(1)
    kw = _thresholds(low, iou, (H, W), rs)
    dec = _Decoder(low, iou)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    a = _gen(sam, _inputs(case), min_mask_region_area=100, **GRID, **kw)[0]
    for budget in (1, 3 * (32 + 4 * ((H + 1) // 2) * ((W + 1) // 2))):      # one mask, three masks per launch
        monkeypatch.setattr(mg, "SMALL_REGIONS_WORKSPACE_BYTES", budget)
        dec.served = 0
        b = _gen(sam, _inputs(case), min_mask_region_area=100, **GRID, **kw)[0]
        for key in KEYS:
            assert _same(a[key], b[key]), (budget, key)


def test_area_zero_is_the_call_without_it(sam):
    img = _image((333, 517), 4)
    kw = dict(points_per_side=6, pred_iou_thresh=0.0, stability_score_thresh=0.0, output_rle_mask=True)
    a = _gen(sam, dict(images=img), **kw)[0]
    for area in (0, 0.0, -5):
        b = _gen(sam, dict(images=img), min_mask_region_area=area, **kw)[0]
        assert a["masks"].shape[0] > 0 and a["rle"] == b["rle"]
        for key in KEYS:
            assert _same(a[key], b[key]), key


def test_two_image_call_equals_single_image_calls(sam, monkeypatch):
    imgs = [_image((600, 800), 2), _image((333, 517), 3)]
    lows, ious = zip(*(_structured(s) for s in (5, 6)))
    kw = dict(points_per_side=N_SIDE, points_per_batch=48, pred_iou_thresh=0.5, stability_score_thresh=0.0,
              crops_nms_thresh=0.5, min_mask_region_area=120)
    both = _Decoder(torch.cat(lows), torch.cat(ious))
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", both)
    res2 = _gen(sam, dict(images=imgs), **kw)
    assert both.served == 2 * N_PTS
    for b, img in enumerate(imgs):
        monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", _Decoder(lows[b], ious[b]))
        r1 = _gen(sam, dict(images=img), **kw)[0]
        assert r1["masks"].shape[0] > 0
        for key in KEYS:
            assert _same(r1[key], res2[b][key]), (b, key)


def test_rle_strings_decode_to_the_cleaned_bits(sam, monkeypatch):
    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.results import coco_rle_to_mask
    case = "u8_600x800"
    (H, W), rs = CASES[case]
    low, iou = _structured(2)
    kw = _thresholds(low, iou, (H, W), rs)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", _Decoder(low, iou))
    r = _gen(sam, _inputs(case), min_mask_region_area=200, output_rle_mask=True, **GRID, **kw)[0]
    m = mg.masks_to_bool(r).cpu().numpy()
    assert len(r["rle"]) == m.shape[0] > 0
    for rle, mk in zip(r["rle"], m):
        assert rle["size"] == [H, W] and (coco_rle_to_mask(rle) == mk).all()


def _host_syncs(fn) -> int:
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_the_step_adds_exactly_one_host_synchronisation(sam, monkeypatch):
    imgs = [_image((600, 800), 2), _image((333, 517), 3)]
    lows, ious = zip(*(_structured(s) for s in (5, 6)))
    dec = _Decoder(torch.cat(lows), torch.cat(ious))
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    counts = {}
    for area in (0, 120):
        for rle in (False, True):
            def call():
                dec.served = 0
                return _gen(sam, dict(images=imgs), points_per_side=N_SIDE, pred_iou_thresh=0.5,
                            stability_score_thresh=0.0, min_mask_region_area=area, output_rle_mask=rle)
            assert all(r["masks"].shape[0] > 0 for r in call())
            counts[(area, rle)] = _host_syncs(call)
    assert counts[(120, False)] == counts[(0, False)] + 1 == 2, counts
    assert counts[(120, True)] == counts[(0, True)] + 1 == 4, counts


def test_no_kept_mask_adds_no_host_synchronisation(sam):
    """With nothing kept there is nothing to clean: the step returns before any device work."""
    img = _image((333, 517), 5)
    counts = {}
    for area in (0, 120):
        def call():
            r = _gen(sam, dict(images=img), points_per_side=4, pred_iou_thresh=1.0, stability_score_thresh=1.0,
                     min_mask_region_area=area)
            assert r[0]["masks"].shape[0] == 0
        call()
        counts[area] = _host_syncs(call)
    assert counts[0] == counts[120] == 1, counts


def test_cli_flag_writes_the_api_dicts(sam, tmp_path):
    import cv2

    from rsprompter_b200 import mask_generation as mg
    rgb = _image((240, 320), 9)
    path = tmp_path / "img.png"
    cv2.imwrite(str(path), rgb.permute(1, 2, 0).flip(-1).numpy())
    ckpt = tmp_path / "sam.pth"
    torch.save(sam["sd"], ckpt)
    out = tmp_path / "masks.json"
    mg.main([str(path), "--arch", "base", "--checkpoint", str(ckpt), "--points-per-side", "4",
             "--pred-iou-thresh", "0", "--stability-score-thresh", "0", "--min-mask-region-area", "500",
             "--out", str(out)])
    rows = json.loads(out.read_text())
    ref = _gen(sam, dict(images=rgb), points_per_side=4, pred_iou_thresh=0.0, stability_score_thresh=0.0,
               min_mask_region_area=500, output_rle_mask=True)[0]
    assert len(rows) > 0 and rows == json.loads(json.dumps(mg.mask_dicts(ref)))
