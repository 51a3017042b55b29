"""Segment-everything over a whole scene on the GPU (ViT-B synthetic weights, seeded as in test_mask_generation_gpu.py):
rsp_sam_mask_stats with the crop-edge rule against it without and the oracle's crop-edge rule; generate_scene_masks on one window
against generate_masks; on six windows against oracle.restate_scene_mask_generation, with structured decoder outputs
and end to end; batch-size invariance, host synchronisations, the refusals and the CLI."""
import json
import warnings

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SCENE = (1536, 2048)         # six 1024 x 1024 windows at the default overlap


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


def _same(a, b) -> bool:
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("crop_box", [(0, 0, 320, 256), (300, 0, 620, 256), (680, 200, 1000, 456), (680, 344, 1000, 600)])
def test_crop_stats_kernel_is_the_stats_kernel_plus_the_edge_rule(crop_box):
    """Masks drawn at the window's own resolution (an identity resize), rectangles whose sides sit 19 to 22 px from each
    window side, and smooth fields; windows of a 600 x 1000 scene: a corner, a top middle, a right edge and the
    bottom-right one."""
    from oracle import restate_scene_mask_generation as O
    from rsprompter_b200 import _lib
    hw = (600, 1000)
    x0, y0, x1, y1 = crop_box
    h, w = y1 - y0, x1 - x0
    maps = []
    for d in (19, 20, 21, 22):
        for side in range(4):
            m = torch.full((h, w), -5.0)
            ys, xs = [100, 140], [100, 140]
            if side == 0:
                xs = [d, 140]
            elif side == 1:
                ys = [d, 140]
            elif side == 2:
                xs = [100, w - d]
            else:
                ys = [100, h - d]
            m[ys[0]:ys[1] + 1, xs[0]:xs[1] + 1] = 5.0
            maps.append(m)
    maps.append(torch.full((h, w), -5.0))                                  # empty: box [0, 0, 0, 0]
    g = torch.Generator().manual_seed(sum(crop_box))
    maps.append(torch.full((h, w), 5.0))
    field = F.interpolate(torch.randn(1, 24, 5, 5, generator=g) * 6, (h, w), mode="bilinear", align_corners=False)[0]
    maps = torch.cat([torch.stack(maps), field]).contiguous().cuda()
    n = maps.shape[0]
    iou = torch.rand(n, generator=g).cuda()
    geom = ((h, w), (h, w), (h, w))
    for pred, stab in ((0.0, 0.0), (0.3, 0.5)):
        a = _lib.sam_mask_stats(maps, geom, 0.0, 1.0, iou, pred, stab)
        b = _lib.sam_mask_stats(maps, geom, 0.0, 1.0, iou, pred, stab, crop=(crop_box, hw))
        for x, y in zip(a[:3], b[:3]):
            assert _same(x.cpu(), y.cpu())
        near = O.near_crop_edge(a[1].cpu().long(), crop_box, hw)
        assert torch.equal(b[3].cpu(), a[3].cpu() & ~near)
        assert 0 < int(near.sum()) < n


# ------------------------------------------------------------------------------------------------ one window
@pytest.mark.parametrize("hw", [(1024, 1024), (600, 800)])
def test_one_window_scene_is_generate_masks(sam, hw):
    from rsprompter_b200 import mask_generation as mg
    img = _image(hw, 1)
    kw = dict(points_per_side=8, points_per_batch=32, pred_iou_thresh=0.0, stability_score_thresh=0.0)
    ref = mg.generate_masks(sam["model"], img, output_rle_mask=True, **kw)[0]
    hwc = img.permute(1, 2, 0).contiguous().permute(2, 0, 1)                # a permuted HWC array
    got = sam["model"].generate_scene_masks(hwc, **kw)
    assert len(got["rle"]) == ref["scores"].shape[0] > 0
    assert [r["counts"] for r in got["rle"]] == [r["counts"] for r in ref["rle"]]
    assert all(r["size"] == list(hw) for r in got["rle"])
    for k in ("scores", "stability_scores", "boxes", "points"):
        assert _same(got[k], ref[k]), k
    assert torch.equal(got["candidates"], ref["candidates"])
    assert got["tiles"].eq(0).all() and got["crop_boxes"].cpu().eq(torch.tensor([0, 0, hw[1], hw[0]])).all()
    assert got["size"] == hw


# ------------------------------------------------------------------------------------------------ six windows
N_SIDE = 6
N_PTS = N_SIDE * N_SIDE


def _blobs(n_tiles, seed):
    """Per window and prompt, 3 low-res fields each holding one blob (a Gaussian bump of random centre and radius,
    over a negative floor): blobs anywhere in the window, so masks cross seams, touch interior and scene edges and
    lie inside the overlaps; tie-free scores."""
    g = torch.Generator().manual_seed(seed)
    n = n_tiles * N_PTS * 3
    cy, cx = torch.rand(n, generator=g) * 300 - 22, torch.rand(n, generator=g) * 300 - 22
    r = 4 + 40 * torch.rand(n, generator=g)
    yy = torch.arange(256.0)[None, :, None]
    xx = torch.arange(256.0)[None, None, :]
    d2 = (yy - cy[:, None, None]) ** 2 + (xx - cx[:, None, None]) ** 2
    low = 12 * torch.exp(-d2 / (2 * r[:, None, None] ** 2)) - 4 + 1e-2 * torch.randn(n, 256, 256, generator=g)
    iou = torch.rand(n_tiles * N_PTS, 3, generator=g)
    return low.view(n_tiles * N_PTS, 3, 256, 256).contiguous(), iou


class _Decoder:
    """Serves seeded outputs in place of the mask decoder, prompt by prompt across windows in slice order."""

    def __init__(self, low, iou):
        self.low, self.iou, self.served = low.cuda(), iou.cuda(), 0

    def __call__(self, emb_rows, pos_rows, sparse, hw, **kw):
        q0 = self.served
        self.served += sparse.shape[0]
        return self.low[q0:self.served], self.iou[q0:self.served]


def _oracle(low, iou, hw, crops, kw, area=0.0):
    from oracle import restate_mask_generation as R
    from oracle import restate_scene_mask_generation as O
    from rsprompter_b200.mask_generation import preprocess_shape
    wins, pts = [], []
    for t, cb in enumerate(crops):
        whw = (cb[3] - cb[1], cb[2] - cb[0])
        sl = slice(t * N_PTS, (t + 1) * N_PTS)
        wins.append(O.generate_window(low[sl], iou[sl], cb, hw, preprocess_shape(whw, 1024),
                                      min_mask_region_area=area, **kw))
        pts.append(R.grid_prompts(N_SIDE, whw)[0])
    return wins, O.merge(wins, crops, pts, kw["crops_nms_thresh"])


def _check_against_oracle(got, merged, wins, crops, hw, low):
    from oracle import restate_mask_generation as R
    from oracle import restate_scene_mask_generation as O
    from rsprompter_b200.mask_generation import preprocess_shape
    from rsprompter_b200.results import coco_rle_to_mask
    assert torch.equal(got["tiles"].cpu(), merged["tiles"])
    assert torch.equal(got["candidates"], merged["candidates"])
    assert torch.equal(got["scores"].cpu(), merged["scores"])
    assert torch.equal(got["boxes"].cpu(), merged["boxes"]) and got["boxes"].dtype == torch.int64
    assert torch.equal(got["points"].cpu(), merged["points"])
    assert _same(got["crop_boxes"].cpu(), torch.tensor(crops)[merged["tiles"]])
    assert torch.allclose(got["stability_scores"].cpu(), merged["stability"], rtol=1e-3, atol=0, equal_nan=True)
    eps = 1e-4 * max(1.0, low.abs().max().item())
    for i, (t, rank, c) in enumerate(zip(merged["tiles"].tolist(), merged["rank"].tolist(),
                                         merged["candidates"].tolist())):
        cb = crops[t]
        whw = (cb[3] - cb[1], cb[2] - cb[0])
        v = R.upscale(low[t * N_PTS + c // 3, c % 3], whw, preprocess_shape(whw, 1024))
        tie = O.uncrop(((v - 0.0).abs() <= eps)[None], cb, hw)[0]
        ref = O.uncrop(wins[t]["masks"][rank][None], cb, hw)[0]
        assert got["rle"][i]["size"] == list(hw)
        m = torch.from_numpy(coco_rle_to_mask(got["rle"][i])).bool()
        assert torch.equal(m & ~tie, ref & ~tie), i


def _kw(low, iou, crops, hw):
    """Thresholds at which the IoU filter, the stability filter, the edge rule and both NMS stages each remove some
    candidates and keep some."""
    from oracle import restate_mask_generation as R
    from rsprompter_b200.mask_generation import preprocess_shape
    cb = crops[1]
    whw = (cb[3] - cb[1], cb[2] - cb[0])
    st = R.mask_stats(R.upscale(low[N_PTS:2 * N_PTS], whw, preprocess_shape(whw, 1024)).flatten(0, 1), 0.0, 1.0)
    v = torch.unique(iou.flatten().double())
    pred = float((v[len(v) // 5] + v[len(v) // 5 + 1]) / 2)
    s = torch.unique(st["stability"][torch.isfinite(st["stability"])].double())
    stab = float((s[len(s) // 10] + s[len(s) // 10 + 1]) / 2)
    return dict(pred_iou_thresh=pred, stability_score_thresh=stab, stability_score_offset=1.0, mask_threshold=0.0,
                crops_nms_thresh=0.5)


@pytest.fixture(scope="module")
def blobs():
    from rsprompter_b200.mask_generation import scene_crop_boxes
    crops = scene_crop_boxes(SCENE, 1024, 0.25)
    assert len(crops) == 6
    low, iou = _blobs(len(crops), seed=5)
    return dict(low=low, iou=iou, crops=crops, kw=_kw(low, iou, crops, SCENE), scene=_image(SCENE, 3))


def _run(sam, monkeypatch, blobs, **kw):
    from rsprompter_b200 import mask_generation as mg
    dec = _Decoder(blobs["low"], blobs["iou"])
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    res = mg.generate_scene_masks(sam["model"], blobs["scene"], points_per_side=N_SIDE, points_per_batch=64,
                                  **dict(blobs["kw"], **kw))
    assert dec.served == len(blobs["crops"]) * N_PTS
    return res


@pytest.mark.parametrize("area", [0.0, 150.5])
def test_six_windows_match_the_oracle_at_every_batch_size(sam, monkeypatch, blobs, area):
    from oracle import restate_scene_mask_generation as O
    low, iou, crops, kw = blobs["low"], blobs["iou"], blobs["crops"], blobs["kw"]
    wins, merged = _oracle(low, iou, SCENE, crops, kw, area)
    # every stage is active: the edge rule drops survivors, and the merge drops some windows' rows and keeps others'
    no_edge = [O.generate_window(low[t * N_PTS:(t + 1) * N_PTS], iou[t * N_PTS:(t + 1) * N_PTS], (0, 0, 1024, 1024),
                                 (1024, 1024), (1024, 1024), **kw) for t in range(len(crops))]
    assert sum(len(w["index"]) for w in no_edge) > sum(len(w["index"]) for w in wins)
    total = sum(len(w["index"]) for w in wins)
    assert 0 < len(merged["tiles"]) < total
    assert len(set(merged["tiles"].tolist())) == len(crops)
    results = [_run(sam, monkeypatch, blobs, batch_size=b, min_mask_region_area=area) for b in (1, 4, 6)]
    _check_against_oracle(results[0], merged, wins, crops, SCENE, low)
    for r in results[1:]:
        assert [x["counts"] for x in r["rle"]] == [x["counts"] for x in results[0]["rle"]]
        for k in ("scores", "stability_scores", "boxes", "points", "tiles", "crop_boxes"):
            assert _same(r[k], results[0][k]), k
        assert torch.equal(r["candidates"], results[0]["candidates"])


def test_six_windows_end_to_end_match_the_oracle(sam):
    """The seeded weights' own decoder outputs for each window, thresholds 0: generate_scene_masks against the oracle
    on the outputs _candidates gives for the same windows."""
    from rsprompter_b200 import mask_generation as mg
    scene = _image(SCENE, 4)
    crops = mg.scene_crop_boxes(SCENE, 1024, 0.25)
    sm = sam["model"].sam_model
    dev = sm.prompt_encoder.no_mask_embed.weight.device
    p = dict(points_per_side=N_SIDE, points_per_batch=64, pred_iou_thresh=0.0, stability_score_thresh=0.0,
             stability_score_offset=1.0, mask_threshold=0.0)
    lows, ious = [], []
    with torch.no_grad():
        for x0, y0, x1, y1 in crops:
            pix, sizes, reshaped = mg._inputs(sm, [scene[:, y0:y1, x0:x1].to(dev)], None, None, None, dev)
            cand = mg._candidates(sm, sm._encode(pix), sizes, reshaped, p)
            lows.append(cand["logits"].view(N_PTS, 3, 256, 256).cpu())
            ious.append(cand["iou"][0].view(N_PTS, 3).cpu())
            del cand
    low, iou = torch.cat(lows), torch.cat(ious)
    kw = dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, stability_score_offset=1.0, mask_threshold=0.0,
              crops_nms_thresh=0.7)
    wins, merged = _oracle(low, iou, SCENE, crops, kw)
    got = mg.generate_scene_masks(sam["model"], scene, points_per_side=N_SIDE, points_per_batch=64, batch_size=4,
                                  **kw)
    _check_against_oracle(got, merged, wins, crops, SCENE, low)


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


@pytest.mark.parametrize("area", [0.0, 150.5])
def test_host_synchronisations_per_batch_and_one_for_the_merge(sam, monkeypatch, blobs, area):
    """generate_masks(output_rle_mask=True)'s count on each batch of windows, and one for the merge, whatever the
    number of kept masks."""
    from rsprompter_b200 import mask_generation as mg
    scene = blobs["scene"].cuda()
    crops = blobs["crops"]
    for b in (2, 3):
        for pred in (blobs["kw"]["pred_iou_thresh"], 0.0):
            kw = dict(blobs["kw"], pred_iou_thresh=pred, points_per_side=N_SIDE, points_per_batch=64,
                      min_mask_region_area=area)

            decoders = iter([_Decoder(blobs["low"], blobs["iou"]) for _ in range(4)])     # built outside the count

            def windows():
                monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", next(decoders))
                return mg.generate_masks(sam["model"], [scene[:, y0:y1, x0:x1] for x0, y0, x1, y1 in crops[:b]],
                                         output_rle_mask=True, **kw)

            def call():
                monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", next(decoders))
                return mg.generate_scene_masks(sam["model"], scene, batch_size=b, **kw)
            assert all(len(r["rle"]) > 0 for r in windows())
            per_batch = _host_syncs(windows)
            res = call()
            assert len(res["rle"]) > 0 and set(res["tiles"].tolist()) == set(range(6)), res["tiles"]
            n = _host_syncs(call)
            assert per_batch == 3 + (area > 0)                  # kept counts; RLE pool size and strings; small regions
            assert n == per_batch * (6 // b) + 1, (n, per_batch, b, pred)


def test_candidate_bound_and_memory_checks(sam, monkeypatch, blobs):
    from rsprompter_b200 import large_image
    from rsprompter_b200 import mask_generation as mg
    # the batch check: before any window runs
    dec = _Decoder(blobs["low"], blobs["iou"])
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    monkeypatch.setattr(mg, "_free_bytes", lambda dev: 1 << 20)
    with pytest.raises(RuntimeError, match=r"1536 x 2048 scene in batches of 4 windows"):
        mg.generate_scene_masks(sam["model"], blobs["scene"], points_per_side=N_SIDE, batch_size=4, **blobs["kw"])
    assert dec.served == 0
    # the merge workspace: after the windows, before the merge
    calls = []
    monkeypatch.setattr(mg, "_free_bytes", lambda dev: calls.append(dev) or (1 << 40 if len(calls) == 1 else 1))
    with pytest.raises(RuntimeError, match="NMS workspace"):
        _run(sam, monkeypatch, blobs, batch_size=4)
    monkeypatch.setattr(mg, "_free_bytes", lambda dev: 1 << 40)
    monkeypatch.setattr(large_image, "MAX_MERGE_CANDIDATES", 5)
    with pytest.raises(ValueError, match=r"6 windows kept \d+ masks.* at most 5 candidates"):
        _run(sam, monkeypatch, blobs, batch_size=4)
    with pytest.raises(ValueError, match="stack expects each tensor"):
        mg.generate_scene_masks(sam["model"], blobs["scene"], crops_n_layers=1)


def test_cli_scene_mode_writes_scene_masks(sam, monkeypatch, blobs, tmp_path):
    import cv2

    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.results import coco_rle_to_mask
    from rsprompter_b200.sam_decoder import SamMaskDecoderB200
    path = tmp_path / "scene.png"
    cv2.imwrite(str(path), blobs["scene"].permute(1, 2, 0).flip(-1).numpy())        # BGR on disk
    ckpt = tmp_path / "sam.pth"
    torch.save(sam["sd"], ckpt)
    dec = _Decoder(blobs["low"], blobs["iou"])
    monkeypatch.setattr(SamMaskDecoderB200, "decode", lambda self, *a, **kw: dec(*a, **kw))     # the CLI's model
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    out = tmp_path / "masks.json"
    kw = blobs["kw"]
    mg.main([str(path), "--arch", "base", "--checkpoint", str(ckpt), "--points-per-side", str(N_SIDE),
             "--pred-iou-thresh", str(kw["pred_iou_thresh"]), "--stability-score-thresh",
             str(kw["stability_score_thresh"]), "--crops-nms-thresh", str(kw["crops_nms_thresh"]),
             "--patch-size", "1024", "--batch-size", "3", "--out", str(out)])
    rows = json.loads(out.read_text())
    dec.served = 0
    ref = mg.generate_scene_masks(sam["model"], blobs["scene"], points_per_side=N_SIDE, **kw)
    assert len(rows) == len(ref["rle"]) > 0
    for row, r, (x1, y1, x2, y2), cb in zip(rows, ref["rle"], ref["boxes"].tolist(), ref["crop_boxes"].tolist()):
        assert set(row) == {"segmentation", "bbox", "predicted_iou", "stability_score", "point_coords", "crop_box"}
        assert row["segmentation"]["size"] == list(SCENE) and row["segmentation"]["counts"] == r["counts"].decode()
        assert row["bbox"] == [x1, y1, x2 - x1, y2 - y1]
        assert row["crop_box"] == [cb[0], cb[1], cb[2] - cb[0], cb[3] - cb[1]]
        assert coco_rle_to_mask(row["segmentation"]).shape == SCENE
