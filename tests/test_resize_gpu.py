"""The test pipeline's keep-ratio Resize + Pad on the device: rsp_resize_pad_u8 and DetDataPreprocessor
(device_transforms=...) against oracle.restate_resize, predict() of resized images against the host pipeline,
predict_records of resized images against predict(), and large scenes with an explicit patch size against a
composition of the device transforms, predict(), the oracle merge, sahi's shift_masks and the host RLE."""
import json

import numpy as np
import pytest
import torch

from oracle import restate_large_image as oracle_li
from oracle import restate_resize as oracle

pytestmark = pytest.mark.gpu

NUM_CLASSES = 10
MEAN = [123.675, 116.28, 103.53]
STD = [58.395, 57.12, 57.375]
PAD_BGR = (0.406 * 255, 0.456 * 255, 0.485 * 255)
SIZES = [(333, 500), (600, 800), (1000, 999), (3000, 1000), (7, 3), (1, 5), (1024, 700), (2048, 2048)]


def _noise(hw, seed):
    return np.random.default_rng(seed).integers(0, 256, (*hw, 3), dtype=np.uint8)


def _norm_pad(pad, swap):
    p = torch.tensor(pad, dtype=torch.float32)
    p = p.flip(0) if swap else p
    return (p - torch.tensor(MEAN, dtype=torch.float32)) / torch.tensor(STD, dtype=torch.float32)


# ---- kernel -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("swap", [True, False], ids=["bgr_to_rgb", "no_flip"])
def test_resize_pad_kernel_matches_oracle(swap):
    """One launch over a mixed batch: CHW planes and HWC views, sizes down / up / identity, within 0.02 / std of the
    float64 oracle; the padded region is the normalised pad value bit for bit."""
    from rsprompter_b200 import _lib
    imgs = [_noise(hw, i) for i, hw in enumerate(SIZES)]
    views = []
    for i, im in enumerate(imgs):
        t = torch.from_numpy(im).cuda()
        views.append(t.permute(2, 0, 1) if i % 2 else t.permute(2, 0, 1).contiguous())      # HWC view / CHW planes
    sizes = [oracle.rescale_size(hw, (1024, 1024)) for hw in SIZES]
    out = torch.empty(len(imgs), 3, 1024, 1024, device="cuda")
    _lib.resize_pad_u8(views, sizes, out, MEAN, STD, swap, PAD_BGR)
    ref, _ = oracle.pipeline(imgs, (1024, 1024), (1024, 1024), PAD_BGR, MEAN, STD, bgr_to_rgb=swap)
    got = out.cpu().double().numpy()
    tol = 0.02 / min(STD)
    padv = _norm_pad(PAD_BGR, swap)
    for b, (nh, nw) in enumerate(sizes):
        assert np.abs(got[b, :, :nh, :nw] - ref[b, :, :nh, :nw]).max() <= tol, SIZES[b]
        for c in range(3):
            pad = torch.cat([out[b, c, nh:, :].reshape(-1), out[b, c, :nh, nw:].reshape(-1)]).cpu()
            assert torch.equal(pad, torch.full_like(pad, float(padv[c]))), (SIZES[b], c)


@pytest.mark.parametrize("hwc", [False, True], ids=["chw", "hwc"])
def test_identity_size_equals_preprocess_u8(hwc):
    from rsprompter_b200 import _lib
    im = torch.from_numpy(_noise((300, 416), 5)).cuda()
    src = im.permute(2, 0, 1) if hwc else im.permute(2, 0, 1).contiguous()
    a = torch.empty(1, 3, 320, 448, device="cuda")
    _lib.resize_pad_u8([src], [(300, 416)], a, MEAN, STD, True, (0.0, 0.0, 0.0))
    b = torch.empty(3, 320, 448, device="cuda")
    _lib.preprocess_u8(src, b, MEAN, STD, True, float(_norm_pad((0.0, 0.0, 0.0), True)[0]))
    assert torch.equal(a[0, 0], b[0])
    assert torch.equal(a[0, :, :300, :416], b[:, :300, :416])


def test_resize_pad_rejects_a_size_beyond_the_pad():
    from rsprompter_b200 import _lib
    src = torch.zeros(3, 10, 10, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.RspError, match="descriptor"):
        _lib.resize_pad_u8([src], [(20, 10)], torch.empty(1, 3, 16, 16, device="cuda"), MEAN, STD, True, PAD_BGR)


# ---- preprocessor -------------------------------------------------------------------------------------------------
def _dp(size=1024, pad=PAD_BGR):
    from rsprompter_b200.preprocess import DetDataPreprocessor
    dp = DetDataPreprocessor(mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32, device_transforms=[
        dict(type="Resize", scale=(size, size), keep_ratio=True),
        dict(type="Pad", size=(size, size), pad_val=dict(img=pad, masks=0))])
    return dp.cuda()


def test_preprocessor_matches_oracle_pipeline():
    from rsprompter_b200 import _lib
    from rsprompter_b200.registry import DetDataSample
    hws = [(333, 500), (600, 800), (1000, 999), (7, 3)]
    imgs = [_noise(hw, 10 + i) for i, hw in enumerate(hws)]
    chw = [torch.from_numpy(im).permute(2, 0, 1).contiguous() for im in imgs]       # PackDetInputs' layout
    samples = [DetDataSample(metainfo={}) for _ in imgs]
    samples[1].set_metainfo(dict(ori_shape=(600, 800)))
    n0 = _lib.launch_count
    out = _dp()(dict(inputs=chw, data_samples=samples))
    assert _lib.launch_count - n0 == 1
    ref, metas = oracle.pipeline(imgs, (1024, 1024), (1024, 1024), PAD_BGR, MEAN, STD)
    assert np.abs(out["inputs"].cpu().double().numpy() - ref).max() <= 0.02 / min(STD)
    for ds, m in zip(out["data_samples"], metas):
        for k in ("ori_shape", "img_shape", "scale_factor", "pad_shape", "batch_input_shape"):
            assert ds.metainfo[k] == m[k], k
            assert type(ds.metainfo[k][0]) is type(m[k][0]), k


# ---- detectors ----------------------------------------------------------------------------------------------------
_DP = dict(type="DetDataPreprocessor", mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32)


def _model_cfg(kind):
    from rsprompter_b200 import model_configs
    if kind == "anchor":
        cfg = model_configs.anchor_model_cfg("base", NUM_CLASSES, mmpretrain_img_size=512)
    elif kind == "query":
        cfg = model_configs.query_model_cfg("base", NUM_CLASSES, prompt_shape=(20, 5), mmpretrain_img_size=512)
    else:
        cfg = model_configs.maskrcnn_model_cfg("base", NUM_CLASSES)
    return dict(cfg, data_preprocessor=_DP)


_MODELS = {}


def _model(kind):
    if kind not in _MODELS:
        from rsprompter_b200 import synthetic
        from rsprompter_b200.model_configs import SELECT_LAYERS
        from rsprompter_b200.registry import MODELS
        m = MODELS.build(_model_cfg(kind))
        arch = m.backbone.vision_encoder.arch
        if kind == "anchor":
            sd = synthetic.anchor_detector_state_dict(arch, NUM_CLASSES, 0, seed=3, pseudo_neck=True)
        elif kind == "query":
            sd = synthetic.query_detector_state_dict(arch, NUM_CLASSES, 0, nq=20, seed=8, pseudo_neck=True)
        else:
            sd = synthetic.maskrcnn_detector_state_dict(arch, NUM_CLASSES, len(SELECT_LAYERS["base"]), seed=11)
        m.load_state_dict(sd, strict=True)
        _MODELS[kind] = m.cuda()
    return _MODELS[kind]


def _scene(h, w, seed):
    """Seeded BGR image: smooth colour fields with a few bright rectangles (something for the detectors to see)."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([127 + 100 * np.sin(xx / g.uniform(20, 90) + yy / g.uniform(20, 90) + c) for c in range(3)], -1)
    for _ in range(12):
        y, x = int(g.integers(0, max(1, h - 40))), int(g.integers(0, max(1, w - 40)))
        img[y:y + int(g.integers(20, 200)), x:x + int(g.integers(20, 200))] = g.uniform(0, 255, 3)
    img += g.normal(0, 8, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def _iou(a, b):
    lt = torch.maximum(a[:, None, :2], b[None, :, :2])
    rb = torch.minimum(a[:, None, 2:], b[None, :, 2:])
    inter = (rb - lt).clamp(min=0).prod(-1)
    area = lambda x: (x[:, 2] - x[:, 0]).clamp(min=0) * (x[:, 3] - x[:, 1]).clamp(min=0)  # noqa: E731
    return inter / (area(a)[:, None] + area(b)[None, :] - inter + 1e-9)


def _matched_fraction(gb, gl, rb, rl, thr=0.9):
    """Greedy one-to-one matching (same label, box IoU >= thr), as the end-to-end tests match detections."""
    if gb.numel() == 0 or rb.numel() == 0:
        return 1.0 if gb.numel() == rb.numel() else 0.0
    iou = _iou(gb, rb)
    iou[gl[:, None] != rl[None, :]] = 0
    n = 0
    for i in iou.max(dim=1).values.argsort(descending=True).tolist():
        j = int(iou[i].argmax())                    # best partner not taken yet (duplicate boxes are common)
        if iou[i, j] >= thr:
            iou[:, j] = -1
            n += 1
    return n / max(gb.shape[0], rb.shape[0])


def _host_batch(model, imgs):
    """The host pipeline: the oracle's float64 resize + pad + normalisation, and the metainfo Resize / Pad write."""
    from rsprompter_b200.registry import DetDataSample
    S = model.backbone.vision_encoder.arch.image_size
    x, metas = oracle.pipeline(imgs, (S, S), (S, S), PAD_BGR, MEAN, STD)
    return torch.from_numpy(x).float().cuda(), [DetDataSample(metainfo=m) for m in metas]


def _device_batch(model, imgs):
    S = model.backbone.vision_encoder.arch.image_size
    chw = [torch.from_numpy(im).permute(2, 0, 1).contiguous() for im in imgs]
    out = _dp(S)(dict(inputs=chw))
    return out["inputs"], out["data_samples"]


@pytest.mark.parametrize("kind", ["anchor", "query"])
def test_predict_of_resized_images_matches_host_pipeline(kind):
    model = _model(kind)
    imgs = [_scene(300, 400, 1), _scene(700, 512, 2)]
    x, ds = _device_batch(model, imgs)
    xr, dr = _host_batch(model, imgs)
    model.test_cfg["rle_masks"] = False
    got = model.predict(x, ds)
    ref = model.predict(xr, dr)
    for g, r, im in zip(got, ref, imgs):
        gp, rp = g.pred_instances, r.pred_instances
        assert rp.bboxes.shape[0] > 0
        assert _matched_fraction(gp.bboxes.cpu(), gp.labels.cpu(), rp.bboxes.cpu(), rp.labels.cpu()) >= 0.8
        assert tuple(gp.masks.shape[1:]) == im.shape[:2]
    model.test_cfg["rle_masks"] = True
    try:
        x, ds = _device_batch(model, imgs)
        got = model.predict(x, ds)
    finally:
        model.test_cfg["rle_masks"] = False
    for g, im in zip(got, imgs):
        assert all(m["size"] == list(im.shape[:2]) for m in g.pred_instances.masks)


@pytest.mark.parametrize("kind", ["anchor", "query", "maskrcnn"])
def test_predict_records_of_resized_images_equal_predict(kind):
    from rsprompter_b200 import _lib
    model = _model(kind)
    imgs = [_scene(300, 400, 3), _scene(300, 400, 4)]
    x, ds = _device_batch(model, imgs)
    rec = model.predict_records(x, batch_data_samples=ds)
    assert rec.hw == (300, 400)
    ref = model.predict(x, ds)
    counts = rec.counts.tolist()
    for b, r in enumerate(ref):
        p = r.pred_instances
        n = p.scores.numel()
        assert n > 0
        rows = rec.rows[b]
        assert counts[b] == n
        assert torch.equal(rows[:n, :4], p.bboxes)
        assert torch.equal(rows[:n, 4], p.scores)
        assert torch.equal(rows[:n, 5].long(), p.labels)
        assert torch.equal(rec.mask_bits[b, :n], _lib.pack_mask_bits(p.masks.contiguous()))


def test_predict_records_rejects_mixed_original_sizes():
    model = _model("anchor")
    x, ds = _device_batch(model, [_scene(300, 400, 5), _scene(320, 400, 6)])
    with pytest.raises(ValueError, match="ori_shape"):
        model.predict_records(x, batch_data_samples=ds)


# ---- large scenes -------------------------------------------------------------------------------------------------
def _composition(model, scene, P, ratio=0.25, iou_thr=0.25, batch_size=8):
    """tiles -> device_transforms -> predict() -> oracle merge -> shift_masks -> host RLE."""
    from rsprompter_b200.results import mask_to_coco_rle
    H, W = scene.shape[:2]
    S = model.backbone.vision_encoder.arch.image_size
    dp = _dp(S, pad=tuple(reversed(MEAN)))           # pad with the mean: 0 after normalisation
    org = oracle_li.slice_origins((H, W), P, ratio)
    tiles, offs = [], []
    for i in range(0, len(org), batch_size):
        chunk = org[i:i + batch_size]
        pad = chunk + [chunk[-1]] * (min(batch_size, len(org)) - len(chunk))
        chw = [torch.from_numpy(scene[y0:y0 + P, x0:x0 + P]).permute(2, 0, 1).contiguous() for x0, y0 in pad]
        out = dp(dict(inputs=chw))
        res = model.predict(out["inputs"], out["data_samples"])
        for r in res[:len(chunk)]:
            p = r.pred_instances
            tiles.append(dict(bboxes=p.bboxes.cpu(), scores=p.scores.cpu(), labels=p.labels.cpu(), masks=p.masks.cpu()))
        offs += chunk
    boxes_only = [{k: t[k] for k in ("bboxes", "scores", "labels")} for t in tiles]
    merged, keep = oracle_li.merge_results_by_nms(boxes_only, offs, (H, W), iou_thr, patch=P)
    masks = [m for t in tiles for m in t["masks"]]
    tile_of = [i for i, t in enumerate(tiles) for _ in range(t["masks"].shape[0])]
    rles = [mask_to_coco_rle(oracle_li.shift_masks(masks[k][None], offs[tile_of[k]], (H, W))[0])["counts"]
            for k in keep.tolist()]
    return merged, rles


def _assert_equal_to_composition(ds, ref, rles, hw):
    p = ds.pred_instances
    assert len(rles) > 0
    assert torch.equal(p.bboxes.cpu(), ref["bboxes"])
    assert torch.equal(p.scores.cpu(), ref["scores"])
    assert torch.equal(p.labels.cpu(), ref["labels"])
    assert [m["counts"] for m in p.masks] == rles
    assert all(m["size"] == list(hw) for m in p.masks)


@pytest.mark.parametrize("kind, P", [("anchor", 320), ("query", 320), ("query", 700), ("maskrcnn", 700)])
def test_patch_size_equals_composition(kind, P):
    from rsprompter_b200.large_image import predict_large_image
    model = _model(kind)
    scene = _scene(1100, 1500, seed=1)
    ds = predict_large_image(model, scene, patch_size=P)
    ref, rles = _composition(model, scene, P)
    _assert_equal_to_composition(ds, ref, rles, (1100, 1500))


def test_scene_smaller_than_patch_is_upscaled():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("anchor")
    scene = _scene(300, 400, seed=3)
    ds = predict_large_image(model, scene, patch_size=640, batch_size=2)
    ref, rles = _composition(model, scene, 640, batch_size=2)
    _assert_equal_to_composition(ds, ref, rles, (300, 400))


def test_patch_size_of_the_model_size_is_the_unresized_path():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("anchor")
    scene = _scene(700, 900, seed=6)
    a = predict_large_image(model, scene).pred_instances
    b = predict_large_image(model, scene, patch_size=512).pred_instances
    assert len(a.masks) > 0
    assert torch.equal(a.bboxes, b.bboxes) and torch.equal(a.scores, b.scores) and a.masks == b.masks


def test_patch_size_cuda_graphs_on_and_off_agree():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("query")
    scene = _scene(700, 1300, seed=4)
    off = predict_large_image(model, scene, batch_size=4, patch_size=320).pred_instances
    model.enable_cuda_graphs()
    try:
        on = predict_large_image(model, scene, batch_size=4, patch_size=320).pred_instances
        again = predict_large_image(model, scene, batch_size=4, patch_size=320).pred_instances
        assert len(model._graphs) == 1
    finally:
        model.enable_cuda_graphs(False)
    for r in (on, again):
        for k in ("bboxes", "scores", "labels"):
            assert torch.equal(getattr(r, k), getattr(off, k)), k
        assert r.masks == off.masks


def test_cli_patch_size_writes_the_result_json(tmp_path):
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
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(out), "--patch-size", "320"])
    got = json.loads(out.read_text())
    ref = coco_results(predict_large_image(model, scene, patch_size=320))
    assert len(ref) > 0 and got == json.loads(json.dumps(ref))
