"""Large-scene inference on the device (rsprompter_b200.large_image): the placed RLE encoder against
results.mask_to_coco_rle of the full canvas, the cross-tile merge against oracle.restate_large_image, and
predict_large_image end to end against a reference composition of predict_records + the oracle merge + sahi's
shift_masks + the host RLE."""
import json

import numpy as np
import pytest
import torch

from oracle import restate_large_image as oracle

pytestmark = pytest.mark.gpu

NUM_CLASSES = 10


def _blobs(n, h, w, seed):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = np.zeros((n, h, w), dtype=bool)
    for i in range(n):
        for _ in range(3):
            cy, cx = g.uniform(0, h), g.uniform(0, w)
            ry, rx = g.uniform(1, max(2, h / 3)), g.uniform(1, max(2, w / 3))
            out[i] |= ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
    return out


def _pixel(P, idx):
    m = np.zeros((P, P), dtype=bool)
    m.reshape(-1)[idx] = True
    return m


# ---- placed RLE ---------------------------------------------------------------------------------------------------
_P = 64
_B = _blobs(4, _P, _P, 0)
_NOISE = np.random.default_rng(1).random((_P, _P)) < 0.5
PLACED = {   # tile [P, P], canvas (H, W), origin (y0, x0)
    "origin": (_B[0], (200, 300), (0, 0)),
    "bottom_right": (_B[1], (200, 300), (136, 236)),
    "full_height_middle": (_NOISE, (64, 300), (0, 100)),          # runs cross canvas columns
    "full_height_first": (_B[2], (64, 300), (0, 0)),
    "full_height_last": (np.ones((_P, _P), bool), (64, 300), (0, 236)),
    "full_canvas": (_NOISE, (64, 64), (0, 0)),
    "ones": (np.ones((_P, _P), bool), (200, 300), (70, 90)),
    "ones_at_bottom": (np.ones((_P, _P), bool), (200, 300), (136, 90)),
    "zeros": (np.zeros((_P, _P), bool), (200, 300), (70, 90)),
    "zeros_full_height": (np.zeros((_P, _P), bool), (64, 300), (0, 90)),
    "first_pixel": (_pixel(_P, 0), (200, 300), (70, 90)),
    "last_pixel": (_pixel(_P, -1), (200, 300), (70, 90)),
    "last_pixel_at_corner": (_pixel(_P, -1), (200, 300), (136, 236)),
    "overhang_rows": (_B[3], (40, 300), (0, 50)),                  # h' = 40 < P: clipped, and full height
    "overhang_cols": (_NOISE, (200, 30), (20, 0)),
    "overhang_both": (np.ones((_P, _P), bool), (33, 45), (0, 0)),
    "w_not_multiple_of_8": (_B[0], (203, 301), (139, 237)),
    "w_not_multiple_of_8_inner": (_NOISE, (203, 301), (17, 101)),
}


def _canvas(tile, hw, yx):
    H, W = hw
    y0, x0 = yx
    h, w = min(tile.shape[0], H - y0), min(tile.shape[1], W - x0)
    c = np.zeros((H, W), dtype=bool)
    c[y0:y0 + h, x0:x0 + w] = tile[:h, :w]
    return c, (h, w)


def _encode_placed(cases, packed):
    """One placed-RLE call over every (tile, canvas, origin) in ``cases`` (tiles of one size)."""
    from rsprompter_b200 import _lib
    tiles = torch.from_numpy(np.stack([t for t, _, _ in cases])).cuda()
    P = tiles.shape[1]
    src = _lib.pack_mask_bits(tiles) if packed else tiles
    ld = src.shape[2]
    pl = []
    for j, (t, (H, W), (y0, x0)) in enumerate(cases):
        pl.append((j * P * ld, ld, P, min(P, H - y0), min(P, W - x0), H, W, y0, x0))
    return _lib.mask_rle_placed([(src, pl)], packed=packed)


@pytest.mark.parametrize("packed", [False, True], ids=["bool", "bits"])
@pytest.mark.parametrize("name", list(PLACED))
def test_placed_rle_equals_canvas_rle(name, packed):
    from rsprompter_b200.results import mask_to_coco_rle
    tile, hw, yx = PLACED[name]
    ref = mask_to_coco_rle(_canvas(tile, hw, yx)[0])["counts"]
    assert _encode_placed([PLACED[name]], packed) == [ref]


@pytest.mark.parametrize("packed", [False, True], ids=["bool", "bits"])
def test_placed_rle_one_call_mixes_canvases_and_repeats(packed):
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import mask_to_coco_rle
    cases = list(PLACED.values())
    ref = [mask_to_coco_rle(_canvas(t, hw, yx)[0])["counts"] for t, hw, yx in cases]
    a = _encode_placed(cases, packed)
    assert a == ref
    assert _encode_placed(cases, packed) == a
    # two groups: tiles of another size (61 wide: W % 8 != 0 in the source too) in the same call
    t61 = _blobs(2, 61, 61, 7)
    canv = [((100, 170), (39, 109)), ((61, 500), (0, 3))]
    src = torch.from_numpy(t61).cuda()
    s2 = _lib.pack_mask_bits(src) if packed else src
    ld = s2.shape[2]
    pl2 = [(j * 61 * ld, ld, 61, min(61, H - y0), min(61, W - x0), H, W, y0, x0)
           for j, ((H, W), (y0, x0)) in enumerate(canv)]
    tiles = torch.from_numpy(np.stack([t for t, _, _ in cases])).cuda()
    s1 = _lib.pack_mask_bits(tiles) if packed else tiles
    ld1 = s1.shape[2]
    pl1 = [(j * _P * ld1, ld1, _P, min(_P, H - y0), min(_P, W - x0), H, W, y0, x0)
           for j, (_, (H, W), (y0, x0)) in enumerate(cases)]
    got = _lib.mask_rle_placed([(s2, pl2), (s1, pl1)], packed=packed)
    ref2 = [mask_to_coco_rle(_canvas(t, hw, yx)[0])["counts"] for t, (hw, yx) in zip(t61, canv)]
    assert got == ref2 + ref


def test_placed_rle_large_canvas():
    """A 1024^2 blob tile in a 20 000 x 20 000 scene (400 M canvas pixels, never formed on the device)."""
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import coco_rle_to_mask, mask_to_coco_rle
    tile = _blobs(1, 1024, 1024, 9)[0]
    H = W = 20000
    y0, x0 = 12000, 18976                                         # the right edge column of tiles
    src = _lib.pack_mask_bits(torch.from_numpy(tile[None]).cuda())
    got = _lib.mask_rle_placed([(src, [(0, 128, 1024, 1024, 1024, H, W, y0, x0)])], packed=True)[0]
    canvas, _ = _canvas(tile, (H, W), (y0, x0))
    assert got == mask_to_coco_rle(canvas)["counts"]
    del canvas
    back = coco_rle_to_mask(dict(size=[H, W], counts=got))
    assert np.array_equal(back[y0:y0 + 1024, x0:x0 + 1024], tile) and int(back.sum()) == int(tile.sum())


# ---- cross-tile merge ---------------------------------------------------------------------------------------------
def _records(n_tiles, P, M, seed, batch=4, full=False):
    """Seeded ResultRecords of n_tiles tiles (batch images each, the last one partly used) with distinct scores."""
    from rsprompter_b200.results import ResultRecord
    g = torch.Generator().manual_seed(seed)
    recs = []
    n_rec = (n_tiles + batch - 1) // batch
    scores = (torch.randperm(n_rec * batch * M, generator=g).float() + 1) / (n_rec * batch * M + 1)
    for r in range(n_rec):
        rec = ResultRecord(batch, M, (P, P), device="cuda")
        xy = torch.rand(batch, M, 2, generator=g) * (P - 8)
        wh = 4 + torch.rand(batch, M, 2, generator=g) * (P / 3)
        b = torch.cat([xy, torch.minimum(xy + wh, torch.full_like(xy, float(P)))], dim=2)
        lab = torch.randint(0, NUM_CLASSES, (batch, M), generator=g).float()
        s = scores[r * batch * M:(r + 1) * batch * M].view(batch, M)
        rec.rows.copy_(torch.cat([b, s[..., None], lab[..., None]], dim=2))
        cnt = torch.full((batch,), M, dtype=torch.int32) if full else torch.randint(0, M + 1, (batch,), generator=g,
                                                                                     dtype=torch.int32)
        rec.counts.copy_(cnt)
        recs.append(rec)
    return recs


def _oracle_merge(recs, origins, hw, thr, P):
    tiles, offs, src = [], [], []
    for r, (rec, org) in enumerate(zip(recs, origins)):
        host = rec.to_host(non_blocking=False)
        for b, o in enumerate(org):
            n = int(host.counts[b])
            rows = host.rows[b, :n]
            tiles.append(dict(bboxes=rows[:, :4], scores=rows[:, 4], labels=rows[:, 5].long()))
            offs.append(o)
            src += [(r, b, s) for s in range(n)]
    merged, keep = oracle.merge_results_by_nms(tiles, offs, hw, thr, patch=P)
    return merged, torch.tensor(src, dtype=torch.int64).view(-1, 3)[keep]


@pytest.mark.parametrize("n_tiles, hw, full", [(1, (512, 512), False), (4, (900, 700), False),
                                               (12, (1100, 1500), False), (130, (4000, 6000), True)],
                         ids=["1", "4", "12", "13000_candidates"])
def test_merge_equals_oracle(n_tiles, hw, full):
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    P, M = 512, 100
    org = slice_origins(hw, P, 0.25)[:n_tiles]
    assert len(org) == n_tiles
    recs = _records(n_tiles, P, M, seed=n_tiles, full=full)
    origins = [org[i:i + 4] for i in range(0, n_tiles, 4)]
    if full:
        assert n_tiles * M > 10000                                # mmcv's split_thr: per-class NMS in the oracle
    got = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25)
    ref, src = _oracle_merge(recs, origins, hw, 0.25, P)
    assert got["bboxes"].shape[0] > 0
    assert torch.equal(got["bboxes"].cpu(), ref["bboxes"])
    assert torch.equal(got["scores"].cpu(), ref["scores"])
    assert torch.equal(got["labels"].cpu(), ref["labels"])
    assert torch.equal(got["source"], src)
    if n_tiles >= 12:
        assert got["labels"].unique().numel() == NUM_CLASSES


def test_merge_score_thr_is_a_filter():
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    P, M, hw = 512, 100, (1100, 1500)
    org = slice_origins(hw, P, 0.25)
    recs = _records(len(org), P, M, seed=5)
    origins = [org[i:i + 4] for i in range(0, len(org), 4)]
    full = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25)
    for thr in (0.3, 0.75):
        cut = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25, score_thr=thr)
        k = full["scores"] >= thr
        assert 0 < int(k.sum()) < full["scores"].numel()
        for name in ("bboxes", "scores", "labels"):
            assert torch.equal(cut[name], full[name][k]), name
        assert torch.equal(cut["source"], full["source"][k.cpu()])


# ---- end to end ---------------------------------------------------------------------------------------------------
_DP = dict(type="DetDataPreprocessor", mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], bgr_to_rgb=True,
           pad_size_divisor=32)


def _model_cfg(kind):
    from rsprompter_b200 import model_configs
    if kind == "anchor":
        cfg = model_configs.anchor_model_cfg("base", NUM_CLASSES, mmpretrain_img_size=512)
    elif kind == "query":
        cfg = model_configs.query_model_cfg("base", NUM_CLASSES, prompt_shape=(20, 5), mmpretrain_img_size=512)
    else:
        cfg = model_configs.maskrcnn_model_cfg("base", NUM_CLASSES)
    return dict(cfg, data_preprocessor=_DP)


def _state_dict(kind, arch):
    from rsprompter_b200 import synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    if kind == "anchor":
        return synthetic.anchor_detector_state_dict(arch, NUM_CLASSES, 0, seed=3, pseudo_neck=True)
    if kind == "query":
        return synthetic.query_detector_state_dict(arch, NUM_CLASSES, 0, nq=20, seed=8, pseudo_neck=True)
    return synthetic.maskrcnn_detector_state_dict(arch, NUM_CLASSES, len(SELECT_LAYERS["base"]), seed=11)


def _build(kind):
    from rsprompter_b200.registry import MODELS
    m = MODELS.build(_model_cfg(kind))
    m.load_state_dict(_state_dict(kind, m.backbone.vision_encoder.arch), strict=True)
    return m.cuda()


_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        _MODELS[kind] = _build(kind)
    return _MODELS[kind]


def _scene(h, w, seed):
    """Seeded BGR scene: smooth colour fields with a few bright rectangles (something for the detectors to see)."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([127 + 100 * np.sin(xx / g.uniform(20, 90) + yy / g.uniform(20, 90) + c) for c in range(3)], -1)
    for _ in range(12):
        y, x = int(g.integers(0, h - 40)), int(g.integers(0, w - 40))
        img[y:y + int(g.integers(20, 200)), x:x + int(g.integers(20, 200))] = g.uniform(0, 255, 3)
    img += g.normal(0, 8, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def _reference(model, scene, ratio, iou_thr, batch_size=8):
    """Tiles cut with torch (NCHW batches), predict_records, host records through the oracle merge, shift_masks and
    the host RLE."""
    from rsprompter_b200.results import mask_to_coco_rle
    H, W = scene.shape[:2]
    P = model.backbone.vision_encoder.arch.image_size
    org = oracle.slice_origins((H, W), P, ratio)
    tiles, offs = [], []
    for i in range(0, len(org), batch_size):
        chunk = org[i:i + batch_size]
        pad = chunk + [chunk[-1]] * (min(batch_size, len(org)) - len(chunk))
        x = torch.stack([torch.from_numpy(scene[y0:y0 + P, x0:x0 + P]).permute(2, 0, 1) for x0, y0 in pad])
        x = x.contiguous().cuda()
        x.rsp_norm = model.data_preprocessor._norm3()
        host = model.predict_records(x).to_host(non_blocking=False)
        torch.cuda.synchronize()
        inst = host.instances()
        tiles += inst[:len(chunk)]
        offs += chunk
    boxes_only = [{k: t[k] for k in ("bboxes", "scores", "labels")} for t in tiles]   # masks: only the kept ones
    merged, keep = oracle.merge_results_by_nms(boxes_only, offs, (H, W), iou_thr, patch=P)
    masks = [m for t in tiles for m in t["masks"]]
    tile_of = [i for i, t in enumerate(tiles) for _ in range(t["masks"].shape[0])]
    rles = [mask_to_coco_rle(oracle.shift_masks(masks[k][None], offs[tile_of[k]], (H, W))[0])["counts"]
            for k in keep.tolist()]
    return merged, rles


@pytest.mark.parametrize("kind", ["anchor", "query", "maskrcnn"])
def test_predict_large_image_equals_reference_composition(kind):
    from rsprompter_b200.large_image import predict_large_image
    model = _model(kind)
    scene = _scene(1100, 1500, seed=1)
    ds = predict_large_image(model, scene)
    ref, rles = _reference(model, scene, 0.25, 0.25)
    p = ds.pred_instances
    assert ds.metainfo["ori_shape"] == (1100, 1500) and ds.metainfo["img_shape"] == (1100, 1500)
    assert len(rles) > 0
    assert torch.equal(p.bboxes.cpu(), ref["bboxes"])
    assert torch.equal(p.scores.cpu(), ref["scores"])
    assert torch.equal(p.labels.cpu(), ref["labels"])
    assert [m["counts"] for m in p.masks] == rles
    assert all(m["size"] == [1100, 1500] for m in p.masks)


@pytest.mark.parametrize("kind", ["anchor", "query"])
def test_one_patch_scene_equals_predict(kind):
    from rsprompter_b200.large_image import predict_large_image
    model = _model(kind)
    scene = _scene(512, 512, seed=2)
    ds = predict_large_image(model, scene, merge_iou_thr=1.0)
    x = torch.from_numpy(scene).permute(2, 0, 1)[None].contiguous().cuda()
    x.rsp_norm = model.data_preprocessor._norm3()
    model.test_cfg["rle_masks"] = True
    try:
        ref = model.predict(x)[0].pred_instances
    finally:
        model.test_cfg["rle_masks"] = False
    order = torch.sort(ref.scores, descending=True, stable=True)[1]
    p = ds.pred_instances
    assert len(p.masks) == order.numel() > 0
    assert torch.equal(p.scores, ref.scores[order])
    assert torch.equal(p.bboxes, ref.bboxes[order])
    assert torch.equal(p.labels, ref.labels[order])
    assert [m["counts"] for m in p.masks] == [ref.masks[i]["counts"] for i in order.tolist()]


@pytest.mark.parametrize("kind", ["anchor", "query"])
def test_scene_smaller_than_patch(kind):
    from rsprompter_b200.large_image import predict_large_image
    from rsprompter_b200.results import coco_rle_to_mask
    model = _model(kind)
    H, W = 300, 1300
    ds = predict_large_image(model, _scene(H, W, seed=3), batch_size=2)
    p = ds.pred_instances
    assert len(p.masks) > 0
    b = p.bboxes.cpu()
    assert (b[:, 0] >= 0).all() and (b[:, 1] >= 0).all() and (b[:, 2] <= W).all() and (b[:, 3] <= H).all()
    for m in p.masks:
        assert m["size"] == [H, W] and coco_rle_to_mask(m).shape == (H, W)


def test_cuda_graphs_on_and_off_agree():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("query")
    scene = _scene(700, 1300, seed=4)
    off = predict_large_image(model, scene, batch_size=4).pred_instances
    model.enable_cuda_graphs()
    try:
        on = predict_large_image(model, scene, batch_size=4).pred_instances
        again = predict_large_image(model, scene, batch_size=4).pred_instances
    finally:
        model.enable_cuda_graphs(False)
    for r in (on, again):
        for k in ("bboxes", "scores", "labels"):
            assert torch.equal(getattr(r, k), getattr(off, k)), k
        assert r.masks == off.masks


def test_host_and_device_scene_agree():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("anchor")
    scene = _scene(600, 900, seed=6)
    a = predict_large_image(model, scene).pred_instances
    b = predict_large_image(model, torch.from_numpy(scene).cuda()).pred_instances
    assert torch.equal(a.bboxes, b.bboxes) and a.masks == b.masks


def test_memory_check_refuses_before_running():
    from rsprompter_b200 import _lib
    from rsprompter_b200.large_image import predict_large_image
    model = _model("query")
    n0 = _lib.launch_count
    with pytest.raises(ValueError, match="merge candidates"):
        predict_large_image(model, np.zeros((20000, 20000, 3), np.uint8), overlap_ratio=0.75)
    assert _lib.launch_count == n0


def test_cli_writes_the_result_json(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from rsprompter_b200.large_image import coco_results, main, predict_large_image
    model = _model("query")
    cfg = tmp_path / "cfg.py"
    cfg.write_text("model = " + repr(_model_cfg("query")) + "\n")
    ckpt = tmp_path / "model.pth"
    torch.save(dict(state_dict=model.state_dict()), ckpt)
    scene = _scene(700, 900, seed=7)
    img = tmp_path / "scene.png"
    cv2.imwrite(str(img), scene)
    out = tmp_path / "results.json"
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(out)])
    got = json.loads(out.read_text())
    ref = coco_results(predict_large_image(model, scene))
    assert len(ref) > 0 and got == json.loads(json.dumps(ref))
