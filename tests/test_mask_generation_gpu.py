"""Segment-everything on the GPU (ViT-B synthetic weights, seeded as in test_sam_prompts_gpu.py): rsp_sam_mask_stats
against a float64 restatement of the two resizes and against the bits rsp_mask_paste pastes through them; then
generate_masks end to end against oracle.restate_mask_generation applied to the decoder outputs the GPU produced for the
same grid, its batch and points_per_batch invariance, empty results, RLE strings, host synchronisations and the CLI."""
import json
import warnings

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


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
    """A seeded uint8 RGB image with smooth structure (so masks have regions) and some noise."""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, 8, 8, generator=g) * 255, hw, mode="bilinear", align_corners=False)[0]
    return (base + 20 * torch.rand(3, *hw, generator=g)).clamp(0, 255).to(torch.uint8)


def _logits(n, hm, wm, seed):
    g = torch.Generator().manual_seed(seed)
    field = F.interpolate(torch.randn(1, n, 6, 6, generator=g) * 8, (hm, wm), mode="bilinear", align_corners=False)[0]
    return (field + 1e-2 * torch.randn(n, hm, wm, generator=g)).contiguous()


# (n, hm, wm, (Hb, Wb), reshaped (crop), original (H, W)): a 600 x 800 image, one whose H * W is not a multiple of
# 16, and hm != wm with a non-square intermediate
KERNEL_CASES = [(5, 256, 256, (1024, 1024), (768, 1024), (600, 800)),
                (4, 256, 256, (1024, 1024), (660, 1024), (333, 517)),
                (3, 64, 96, (256, 384), (200, 384), (150, 301))]
BOUND = 1e-4      # |fp32 - fp64| of the two resizes is far below BOUND * max(1, max |logit|)


def _f64(maps, geom):
    (Hb, Wb), (ch, cw), (H, W) = geom
    x = F.interpolate(maps.double()[None], (Hb, Wb), mode="bilinear", align_corners=False)[..., :ch, :cw]
    return F.interpolate(x, (H, W), mode="bilinear", align_corners=False)[0]


def _box(binary):
    n, H, W = binary.shape
    rows, cols = binary.any(-1), binary.any(-2)
    ys, xs = torch.arange(H), torch.arange(W)
    b = torch.stack([torch.where(cols, xs, W).min(-1).values, torch.where(rows, ys, H).min(-1).values,
                     torch.where(cols, xs, -1).max(-1).values, torch.where(rows, ys, -1).max(-1).values], -1)
    return torch.where(binary.flatten(1).any(1)[:, None], b, torch.zeros_like(b))


@pytest.mark.parametrize("case", range(len(KERNEL_CASES)))
@pytest.mark.parametrize("thr, off", [(0.0, 1.0), (0.3, 0.5)])
def test_stats_kernel_matches_float64_resizes(case, thr, off):
    from rsprompter_b200 import _lib
    n, hm, wm, pad, rs, hw = KERNEL_CASES[case]
    maps = _logits(n, hm, wm, seed=case)
    iou = torch.rand(n, generator=torch.Generator().manual_seed(case))
    counts, boxes, stab, keep = _lib.sam_mask_stats(maps.cuda(), (pad, rs, hw), thr, off, iou.cuda(), 0.5, 0.9)
    counts, boxes, stab, keep = counts.cpu(), boxes.cpu(), stab.cpu(), keep.cpu()
    v = _f64(maps, (pad, rs, hw))
    eps = BOUND * max(1.0, maps.abs().max().item())
    for k, t in enumerate((thr + off, thr - off, thr)):
        ref = (v > t).sum((-2, -1))
        ambiguous = ((v - t).abs() <= eps).sum((-2, -1))
        assert ((counts[:, k] - ref).abs() <= ambiguous).all(), (k, counts[:, k], ref, ambiguous)
    sure, possible = _box(v > thr + eps), _box(v > thr - eps)
    assert (boxes[:, :2] <= sure[:, :2]).all() and (boxes[:, 2:] >= sure[:, 2:]).all()
    assert (boxes[:, :2] >= possible[:, :2]).all() and (boxes[:, 2:] <= possible[:, 2:]).all()
    exact = (sure == possible).all(1)
    assert exact.any() and torch.equal(boxes[exact], sure[exact].int())
    # the stability score and the keep flag follow from the counts exactly
    expect = counts[:, 0].float() / counts[:, 1].float()
    assert torch.allclose(stab, expect, rtol=0, atol=0, equal_nan=True)
    assert torch.equal(keep, (iou > 0.5) & (stab > 0.9))


@pytest.mark.parametrize("case", range(len(KERNEL_CASES)))
def test_stats_kernel_agrees_with_pasted_bits(case):
    from rsprompter_b200 import _lib
    n, hm, wm, pad, rs, (H, W) = KERNEL_CASES[case]
    maps = _logits(n, hm, wm, seed=10 + case).cuda()
    counts, boxes, _, keep = _lib.sam_mask_stats(maps, (pad, rs, (H, W)), 0.0, 1.0)
    assert keep is None
    bits = torch.empty(n, H, (W + 15) // 16 * 2, dtype=torch.uint8, device="cuda")
    _lib.mask_paste(maps, 0.0, raw=True, rescale=(pad, rs, (H, W)), bits=bits)
    m = _lib.unpack_mask_bits(bits, bits.shape[2] * 8)[..., :W].cpu()
    assert torch.equal(counts[:, 2].cpu(), m.sum((-2, -1)).int())
    assert torch.equal(boxes.cpu(), _box(m).int())


@pytest.mark.parametrize("pred, stab", [(0.0, 0.0), (0.0, 0.5), (0.5, 0.0), (-1.0, -1.0)])
def test_stats_kernel_threshold_at_or_below_zero_disables_its_test(pred, stab):
    """filter_masks' rule (image_processing_sam.py:350-356): a threshold <= 0 switches its test off, so negative
    scores and the NaN stability of an empty union pass it; an enabled test drops both."""
    from rsprompter_b200 import _lib
    maps = _logits(6, 64, 64, seed=20)
    maps[:2] = -100.0                                    # nothing > thr - offset: 0 / 0 stability
    iou = torch.tensor([-0.5, 0.7, -0.2, 0.9, 0.3, -1.0])
    _, _, st, keep = _lib.sam_mask_stats(maps.cuda(), ((256, 256), (256, 256), (100, 100)), 0.0, 1.0, iou.cuda(),
                                         pred, stab)
    st, keep = st.cpu(), keep.cpu()
    assert st[:2].isnan().all() and st[2:].isfinite().all()
    expect = torch.ones(6, dtype=torch.bool)
    if pred > 0:
        expect &= iou > pred
    if stab > 0:
        expect &= st > stab
    assert torch.equal(keep, expect)
    assert expect.any() and (pred > 0 or stab > 0 or expect.all())


# ------------------------------------------------------------------------------------------------ end to end
def _gen(sam, inputs, **kw):
    from rsprompter_b200 import mask_generation as mg
    return mg.generate_masks(sam["model"], **inputs, **kw)


def _decoder_candidates(sam, inputs, p):
    """The decoder outputs generate_masks filters, for the same grid (its own decode stage)."""
    from rsprompter_b200 import mask_generation as mg
    sm = sam["model"].sam_model
    dev = sm.prompt_encoder.no_mask_embed.weight.device
    with torch.no_grad():
        pix, sizes, reshaped = mg._inputs(sm, inputs.get("images"), inputs.get("pixel_values"),
                                          inputs.get("original_sizes"), inputs.get("reshaped_input_sizes"), dev)
        cand = mg._candidates(sm, sm._encode(pix), sizes, reshaped, dict(p, pred_iou_thresh=0.0,
                                                                           stability_score_thresh=0.0))
    return cand


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


def _inputs(case):
    if case == "u8_1024":
        return dict(images=_image((1024, 1024), 1))
    if case == "u8_600x800":
        return dict(images=[_image((600, 800), 2)])
    g = torch.Generator().manual_seed(3)
    pv = torch.zeros(1, 3, 1024, 1024)
    pv[..., :660, :] = F.interpolate(torch.randn(1, 3, 16, 16, generator=g), (660, 1024), mode="bilinear",
                                     align_corners=False)
    return dict(pixel_values=pv, original_sizes=[(333, 517)], reshaped_input_sizes=[(660, 1024)])


def _compare(got, ref, low, thr, hw, rs, n_side):
    from oracle import restate_mask_generation as R
    from rsprompter_b200 import mask_generation as mg
    H, W = hw
    assert got["size"] == (H, W)
    assert torch.equal(got["candidates"], ref["index"])
    assert torch.equal(got["scores"].cpu(), ref["scores"])
    assert torch.equal(got["boxes"].cpu(), ref["boxes"])
    pts, _ = R.grid_prompts(n_side, (H, W))
    assert torch.equal(got["points"].cpu(), pts[ref["index"] // 3])
    # masks: bit-equal except where the fp32 value sits at the threshold
    m = mg.masks_to_bool(got).cpu()
    v = R.upscale(low, (H, W), rs).flatten(0, 1)[ref["index"]]
    tie = (v - thr).abs() <= BOUND * max(1.0, low.abs().max().item())
    assert torch.equal(m & ~tie, ref["masks"] & ~tie)
    assert torch.allclose(got["stability_scores"].cpu(), ref["stability"], rtol=1e-3, atol=0, equal_nan=True)


@pytest.mark.parametrize("case", ["u8_1024", "u8_600x800", "pixel_values"])
def test_generate_masks_matches_restatement(sam, case):
    """The seeded decoder's masks hardly depend on the prompt (all of them cover the image), so the filters are
    switched off here and the NMS leaves few masks; the stages are exercised on structured decoder outputs below."""
    from oracle import restate_mask_generation as R
    inputs = _inputs(case)
    p = dict(points_per_side=8, points_per_batch=16, stability_score_offset=1.0, mask_threshold=0.0)
    cand = _decoder_candidates(sam, inputs, p)
    H, W = cand["sizes"][0]
    rs = cand["reshaped"][0]
    low = cand["logits"].view(64, 3, 256, 256).cpu()
    iou = cand["iou"][0].view(64, 3).cpu()
    ref = R.generate(low, iou, (H, W), rs, pred_iou_thresh=0.0, stability_score_thresh=0.0, crops_nms_thresh=0.7)
    got = _gen(sam, inputs, pred_iou_thresh=0.0, stability_score_thresh=0.0, crops_nms_thresh=0.7, **p)[0]
    assert ref["after_nms"] > 0
    _compare(got, ref, low, 0.0, (H, W), rs, 8)


@pytest.mark.parametrize("case", ["u8_1024", "u8_600x800", "pixel_values"])
def test_generate_masks_stages_on_structured_decoder_outputs(sam, case, monkeypatch):
    """generate_masks with the decoder replaced by seeded smooth fields per prompt (masks with regions of different
    sizes and places, tie-free scores): thresholds at which the IoU filter, the stability filter and the NMS each
    remove some candidates and keep some, against the restatement on the same outputs."""
    from oracle import restate_mask_generation as R
    inputs = _inputs(case)
    n_side, n_pts = 8, 64
    g = torch.Generator().manual_seed(len(case))
    field = F.interpolate(torch.randn(n_pts, 3, 5, 5, generator=g) * 6, (256, 256), mode="bilinear",
                          align_corners=False)
    low = (field + 1.5 + 1e-2 * torch.randn(n_pts, 3, 256, 256, generator=g)).contiguous()
    iou = torch.rand(n_pts, 3, generator=g)
    served = [0]

    def decode(emb_rows, pos_rows, sparse, hw, **kw):
        q0 = served[0]
        served[0] += sparse.shape[0]
        return low[q0:served[0]].cuda(), iou[q0:served[0]].cuda()

    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", decode)
    sizes = {"u8_1024": (1024, 1024), "u8_600x800": (600, 800), "pixel_values": (333, 517)}
    H, W = sizes[case]
    from rsprompter_b200.mask_generation import preprocess_shape
    rs = (660, 1024) if case == "pixel_values" else preprocess_shape((H, W), 1024)
    st = R.mask_stats(R.upscale(low, (H, W), rs).flatten(0, 1), 0.0, 1.0)
    pred = _between(iou.flatten(), 0.25)
    stab = _between(st["stability"][iou.flatten() > pred], 0.25)
    surv = (iou.flatten() > pred) & (st["stability"] > stab)
    nms = _between(_pairwise_iou(st["boxes"][surv]), 0.7)
    ref = R.generate(low, iou, (H, W), rs, pred_iou_thresh=pred, stability_score_thresh=stab, crops_nms_thresh=nms)
    assert 0 < ref["after_iou"] < ref["candidates"]
    assert 0 < ref["after_stability"] < ref["after_iou"]
    assert 0 < ref["after_nms"] < ref["after_stability"]
    got = _gen(sam, inputs, points_per_side=n_side, points_per_batch=16, pred_iou_thresh=pred,
               stability_score_thresh=stab, crops_nms_thresh=nms)[0]
    assert served[0] == n_pts
    _compare(got, ref, low, 0.0, (H, W), rs, n_side)


CANDIDATE_FIELDS = ("logits", "iou", "stability", "boxes", "keep", "points")


def _candidate_outputs(sam, inputs, n_side, ppb):
    return _decoder_candidates(sam, inputs, dict(points_per_side=n_side, points_per_batch=ppb,
                                                  stability_score_offset=1.0, mask_threshold=0.0))


def test_batch_of_two_gives_each_single_image_result(sam):
    """Candidate for candidate (logits, scores, stability, boxes, keep flags, points), not only the few masks the NMS
    keeps: calls of 48 prompts put both images' prompts in one decoder call, and the encoder runs both at once."""
    imgs = [_image((1024, 1024), 1), _image((600, 800), 2)]
    both = _candidate_outputs(sam, dict(images=imgs), 8, 48)
    for b, img in enumerate(imgs):
        one = _candidate_outputs(sam, dict(images=img), 8, 48)
        nc = one["iou"].shape[1]
        assert torch.equal(one["logits"], both["logits"][b * nc:(b + 1) * nc]), "logits"
        for k in CANDIDATE_FIELDS[1:]:
            assert torch.equal(one[k][0], both[k][b]), k
    kw = dict(points_per_side=8, points_per_batch=48, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    res2 = _gen(sam, dict(images=imgs), **kw)
    for img, r2 in zip(imgs, res2):
        r1 = _gen(sam, dict(images=img), **kw)[0]
        assert r1["masks"].shape[0] > 0
        for k in ("masks", "scores", "stability_scores", "boxes", "points", "candidates"):
            assert torch.equal(r1[k], r2[k]), k


def test_points_per_batch_does_not_change_the_result(sam):
    """1 024 prompts in 16 decoder calls of 64 or in one call of 1 024 (and one stats launch over 3 072 masks): every
    candidate-level output is the same bytes, and so is the (non-empty) result."""
    img = _image((600, 800), 4)
    a = _candidate_outputs(sam, dict(images=img), 32, 64)
    b = _candidate_outputs(sam, dict(images=img), 32, 1024)
    for k in CANDIDATE_FIELDS:
        assert torch.equal(a[k], b[k]), k
    del a, b
    kw = dict(points_per_side=32, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    ra = _gen(sam, dict(images=img), points_per_batch=64, **kw)[0]
    rb = _gen(sam, dict(images=img), points_per_batch=1024, **kw)[0]
    assert ra["masks"].shape[0] > 0
    for k in ("masks", "scores", "stability_scores", "boxes", "points", "candidates"):
        assert torch.equal(ra[k], rb[k]), k


def test_thresholds_of_one_give_empty_results(sam):
    from rsprompter_b200 import mask_generation as mg
    r = _gen(sam, dict(images=_image((333, 517), 5)), points_per_side=4, pred_iou_thresh=1.0,
             stability_score_thresh=1.0, output_rle_mask=True)[0]
    assert r["masks"].shape == (0, 333, 66) and r["masks"].dtype == torch.uint8
    assert r["scores"].shape == (0,) and r["stability_scores"].shape == (0,)
    assert r["boxes"].shape == (0, 4) and r["boxes"].dtype == torch.int64
    assert r["points"].shape == (0, 2) and r["rle"] == [] and r["candidates"].shape == (0,)
    assert mg.masks_to_bool(r).shape == (0, 333, 517)


def test_rle_strings_decode_to_the_bits(sam):
    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.results import coco_rle_to_mask
    r = _gen(sam, dict(images=_image((333, 517), 6)), points_per_side=6, pred_iou_thresh=0.0,
             stability_score_thresh=0.0, output_rle_mask=True)[0]
    m = mg.masks_to_bool(r).cpu().numpy()
    assert len(r["rle"]) == m.shape[0] > 0
    for rle, mk in zip(r["rle"], m):
        assert rle["size"] == [333, 517]
        assert (coco_rle_to_mask(rle) == mk).all()


def _host_syncs(fn) -> int:
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    # the mode's one-time "prototype feature" notice also mentions synchronisation: count only the operations
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_host_synchronisations_do_not_grow_with_the_grid(sam):
    img = _image((600, 800), 7).cuda()
    kw = dict(pred_iou_thresh=0.0, stability_score_thresh=0.0)
    counts = {}
    for n in (4, 16):
        for rle in (False, True):
            def call():
                return _gen(sam, dict(images=img), points_per_side=n, points_per_batch=16, output_rle_mask=rle, **kw)
            call()
            counts[(n, rle)] = _host_syncs(call)
    # the read of the kept counts and candidates, and with RLE the pool size and the strings
    assert counts[(4, False)] == counts[(16, False)] == 1, counts
    assert counts[(4, True)] == counts[(16, True)] == 3, counts


def test_rssam_model_method_is_the_generator(sam):
    img = _image((600, 800), 8)
    a = sam["model"].generate_masks(img, points_per_side=4, pred_iou_thresh=0.0)[0]
    b = _gen(sam, dict(images=img), points_per_side=4, pred_iou_thresh=0.0)[0]
    assert torch.equal(a["masks"], b["masks"]) and torch.equal(a["scores"], b["scores"])


def test_cli_writes_mask_json(sam, tmp_path):
    import cv2

    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.results import coco_rle_to_mask
    rgb = _image((240, 320), 9)
    path = tmp_path / "img.png"
    cv2.imwrite(str(path), rgb.permute(1, 2, 0).flip(-1).numpy())        # BGR on disk
    ckpt = tmp_path / "sam.pth"
    torch.save(sam["sd"], ckpt)
    out = tmp_path / "masks.json"
    mg.main([str(path), "--arch", "base", "--checkpoint", str(ckpt), "--points-per-side", "4",
             "--pred-iou-thresh", "0", "--stability-score-thresh", "0", "--out", str(out)])
    rows = json.loads(out.read_text())
    ref = _gen(sam, dict(images=rgb), points_per_side=4, pred_iou_thresh=0.0, stability_score_thresh=0.0)[0]
    assert len(rows) == ref["masks"].shape[0] > 0
    for row, s, (x1, y1, x2, y2) in zip(rows, ref["scores"].tolist(), ref["boxes"].tolist()):
        assert set(row) == {"segmentation", "bbox", "predicted_iou", "stability_score", "point_coords"}
        assert row["predicted_iou"] == s and row["bbox"] == [x1, y1, x2 - x1, y2 - y1]
        m = coco_rle_to_mask(row["segmentation"])
        assert m.shape == (240, 320) and m.any()
