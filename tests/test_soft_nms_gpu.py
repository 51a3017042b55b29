"""Soft-NMS on the GPU (rsp_soft_nms_batched) against oracle.restate_soft_nms, bit for bit: the kernel on seeded and
constructed problems, the anchor heads with soft RPN / RoI NMS, and the large-scene soft merge."""
import json

import pytest
import torch

from oracle import restate_soft_nms as R

pytestmark = pytest.mark.gpu


def _problem(g, n, n_ids, kind):
    xy = torch.rand(n, 2, generator=g) * 300
    wh = torch.rand(n, 2, generator=g) * 60
    b = torch.cat([xy, xy + wh], 1)
    s = torch.rand(n, generator=g)
    if kind == "ties":                      # duplicate boxes with duplicate scores, coarse scores
        s = torch.round(s * 16) / 16
        k = n // 3
        b[n - k:], s[n - k:] = b[:k], s[:k]
    elif kind == "saturated":
        s[torch.rand(n, generator=g) < 0.5] = 1.0
    elif kind == "zero_area":
        z = torch.rand(n, generator=g) < 0.3
        b[z, 2] = b[z, 0]
        zz = torch.rand(n, generator=g) < 0.2
        b[zz, 3] = b[zz, 1]
    ids = torch.randint(0, n_ids, (n,), generator=g)
    return b.float(), s.float(), ids


def _run(boxes, scores, ids, nvalid, G, cfg, K):
    from rsprompter_b200 import _lib
    return _lib.soft_nms_batched(boxes.cuda().contiguous(), scores.cuda().contiguous(), ids.cuda().contiguous(),
                                 nvalid.int().cuda(), G, cfg["iou_threshold"], cfg["sigma"], cfg["min_score"],
                                 cfg["method"], K=K)


def _same_f32(a, b):
    """Bit-identical fp32, except that any NaN equals any NaN (the device and numpy write different NaN payloads)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def _check_image(out, b, boxes, scores, ids, nv, cfg, K):
    ob, os_, ol, oi, cnt = (t[b].cpu() for t in out)
    dets, keep = R.batched_nms(boxes[:nv], scores[:nv], ids[:nv], dict(type="soft_nms", **cfg))
    k = min(keep.numel(), K)
    assert int(cnt) == k
    assert torch.equal(oi[:k].long(), keep[:k])
    assert torch.equal(ob[:k], dets[:k, :4]) and _same_f32(os_[:k], dets[:k, 4])
    assert torch.equal(ol[:k], ids[keep[:k]])
    assert (oi[k:] == -1).all() and (os_[k:] == 0).all() and (ob[k:] == 0).all()


CFGS = [dict(iou_threshold=0.3, sigma=0.5, min_score=1e-3), dict(iou_threshold=0.5, sigma=0.1, min_score=0.05)]


@pytest.mark.parametrize("method", ["naive", "linear", "gaussian"])
@pytest.mark.parametrize("B,n,G,K,kind,cfg", [
    (1, 1, 1, 0, "random", 0), (3, 7, 2, 0, "ties", 1), (3, 7, 2, 1, "saturated", 0),
    (8, 1000, 10, 100, "random", 0), (8, 1000, 10, 0, "ties", 1), (3, 1000, 3, 1000, "zero_area", 0),
    (1, 8000, 5, 1000, "saturated", 1), (3, 8000, 10, 0, "random", 0),
    (3, 10000, 10, 100, "ties", 0), (1, 10000, 10, 0, "random", 1), (1, 20000, 1, 0, "random", 0),
])
def test_kernel_equals_restatement(method, B, n, G, K, kind, cfg):
    g = torch.Generator().manual_seed(n * 7 + B + K)
    cfg = dict(CFGS[cfg], method=method)
    probs = [_problem(g, n, G, kind) for _ in range(B)]
    boxes = torch.stack([p[0] for p in probs])
    scores = torch.stack([p[1] for p in probs])
    ids = torch.stack([p[2] for p in probs])
    nvalid = torch.tensor([n] + [max(0, n - 3 * i) for i in range(1, B)])
    if B == 8:
        nvalid[5] = 0                                         # an empty problem
    out = _run(boxes, scores, ids, nvalid, G, cfg, K)
    torch.cuda.synchronize()
    for b in range(B):
        _check_image(out, b, boxes[b], scores[b], ids[b], int(nvalid[b]), cfg, K if K > 0 else n)


def test_early_exit_is_a_prefix_of_the_full_run():
    g = torch.Generator().manual_seed(3)
    boxes, scores, ids = _problem(g, 5000, 4, "ties")
    cfg = dict(CFGS[0], method="linear")
    full = _run(boxes[None], scores[None], ids[None], torch.tensor([5000]), 4, cfg, 0)
    part = _run(boxes[None], scores[None], ids[None], torch.tensor([5000]), 4, cfg, 37)
    assert int(part[4][0]) == 37
    for a, b in zip(full[:4], part[:4]):
        assert torch.equal(a[:, :37], b)


def test_bad_arguments_are_refused():
    from rsprompter_b200 import _lib
    x = torch.zeros(1, 4, 4, device="cuda")
    s = torch.zeros(1, 4, device="cuda")
    i = torch.zeros(1, 4, dtype=torch.int64, device="cuda")
    nv = torch.ones(1, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.RspError, match="id groups"):
        _lib.soft_nms_batched(x, s, i, nv, 2000, 0.3)
    with pytest.raises(_lib.RspError, match="sigma"):
        _lib.soft_nms_batched(x, s, i, nv, 1, 0.3, sigma=0.0, method="gaussian")
    with pytest.raises(ValueError, match="method"):
        _lib.soft_nms_batched(x, s, i, nv, 1, 0.3, method="matrix")


# ---- detectors ------------------------------------------------------------------------------------------------------
SOFT = dict(type="soft_nms", iou_threshold=0.5, min_score=0.05)
_MODELS = {}


def _model(kind, C, rpn_soft=False, score_thr=0.05):
    key = (kind, C, rpn_soft, score_thr)
    if key not in _MODELS:
        from rsprompter_b200 import model_configs, synthetic
        from rsprompter_b200.model_configs import SELECT_LAYERS
        from rsprompter_b200.registry import MODELS
        from rsprompter_b200.sam_config import VISION_ARCHS
        if kind == "anchor":
            cfg = model_configs.anchor_model_cfg("base", C)
            sd = synthetic.anchor_detector_state_dict(VISION_ARCHS["base"], C, 6, seed=3)
        else:
            cfg = model_configs.maskrcnn_model_cfg("base", C)
            sd = synthetic.maskrcnn_detector_state_dict(VISION_ARCHS["base"], C, len(SELECT_LAYERS["base"]), seed=11)
        cfg["test_cfg"]["rcnn"]["nms"] = dict(SOFT)
        cfg["test_cfg"]["rcnn"]["score_thr"] = score_thr
        if rpn_soft:
            cfg["test_cfg"]["rpn"]["nms"] = dict(type="soft_nms", iou_threshold=0.7, min_score=0.01,
                                                 method="gaussian", sigma=0.5)
        m = MODELS.build(cfg)
        m.load_state_dict(sd, strict=True)
        _MODELS[key] = m.cuda()
    return _MODELS[key]


def _nhwc_bf16(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()


@pytest.mark.parametrize("kind,C,score_thr", [("anchor", 2, 0.05), ("anchor", 10, 0.0), ("maskrcnn", 10, 0.0)],
                         ids=["anchor_2cls", "anchor_10cls_split", "maskrcnn_10cls_split"])
def test_roi_head_soft_nms_equals_oracle(kind, C, score_thr):
    m = _model(kind, C, score_thr=score_thr)
    g = torch.Generator().manual_seed(7)
    B, K = 2, 1000
    feats = [_nhwc_bf16(torch.randn(B, 256, s, s, generator=g)) for s in (256, 128, 64, 32, 16)]
    ctr = torch.rand(B, K, 2, generator=g) * 1024
    wh = torch.exp(torch.rand(B, K, 2, generator=g) * 5.0 + 1.5)
    props = torch.cat([(ctr - wh / 2).clamp(0, 1024), (ctr + wh / 2).clamp(0, 1024)], dim=2)
    pcnt = torch.tensor([K, K - 123], dtype=torch.int32)
    props[1, K - 123:] = 0
    cap = {}
    if kind == "anchor":
        r = m.roi_head.predict_nhwc(feats, props.cuda(), pcnt.cuda(), (1024, 1024),
                                    torch.randn(B * 4096, 256, generator=g).cuda(),
                                    torch.randn(4096, 256, generator=g).cuda(), (64, 64), capture=cap)
    else:
        r = m.roi_head.predict_nhwc(feats, props.cuda(), pcnt.cuda(), (1024, 1024), capture=cap)
    torch.cuda.synchronize()
    cb, cs, cl = (t.cpu() for t in cap["candidates"])
    split = False
    for b in range(B):
        v = cs[b] >= 0                                          # score > score_thr, (RoI, class) order
        split |= int(v.sum()) >= R.SPLIT_THR
        dets, keep = R.batched_nms(cb[b][v], cs[b][v], cl[b][v], SOFT)
        k = min(keep.numel(), 100)
        assert int(r["counts"][b]) == k > 0
        assert torch.equal(r["bboxes"][b, :k].cpu(), dets[:k, :4])
        assert torch.equal(r["scores"][b, :k].cpu(), dets[:k, 4])
        assert torch.equal(r["labels"][b, :k].cpu(), cl[b][v][keep[:k]])
    assert split == (score_thr == 0.0)


@pytest.mark.parametrize("kind", ["anchor", "maskrcnn"])
def test_rpn_soft_nms_equals_oracle(kind):
    m = _model(kind, 2, rpn_soft=True)
    g = torch.Generator().manual_seed(9)
    feats = [_nhwc_bf16(torch.randn(2, 256, s, s, generator=g)) for s in (256, 128, 64, 32, 16)]
    cap = {}
    pb, ps, cnt = m.rpn_head.predict_nhwc(feats, (1024, 1024), capture=cap)
    torch.cuda.synchronize()
    cb, cs, ci = (t.cpu() for t in cap["candidates"])
    nms = m.rpn_head._nms
    cfg = dict(type="soft_nms", **{k: nms[k] for k in ("iou_threshold", "sigma", "min_score", "method")})
    for b in range(2):
        v = cs[b] >= 0
        rb, rs = R.rpn_nms(cb[b][v], cs[b][v], ci[b][v], cfg, 1000)
        k = int(cnt[b])
        assert k == rb.shape[0] > 0
        assert torch.equal(pb[b, :k].cpu(), rb) and torch.equal(ps[b, :k].cpu(), rs)


@pytest.mark.parametrize("kind,C", [("anchor", 2), ("anchor", 10), ("maskrcnn", 10)])
def test_predict_records_and_cuda_graphs_agree(kind, C):
    m = _model(kind, C, rpn_soft=(C == 2))
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(2, 3, 1024, 1024, generator=g) * 40).cuda()
    preds = m.predict(x.clone())
    rec = m.predict_records(x.clone()).to_host(non_blocking=False)
    for b, ds in enumerate(preds):
        p = ds.pred_instances
        n = int(rec.counts[b])
        assert n == p.scores.numel() > 0
        assert torch.equal(rec.rows[b, :n, :4], p.bboxes.cpu()) and torch.equal(rec.rows[b, :n, 4], p.scores.cpu())
        assert torch.equal(rec.rows[b, :n, 5].long(), p.labels.cpu())
    m.enable_cuda_graphs()
    try:
        g1 = m.predict_records(x.clone()).to_host(non_blocking=False)
        g2 = m.predict_records(x.clone()).to_host(non_blocking=False)
    finally:
        m.enable_cuda_graphs(False)
    for r in (g1, g2):
        assert torch.equal(r.rows, rec.rows) and torch.equal(r.counts, rec.counts)
        assert torch.equal(r.mask_bits, rec.mask_bits)


# ---- large scenes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_tiles, hw, full", [(1, (512, 512), False), (4, (900, 700), False),
                                               (12, (1100, 1500), False), (130, (4000, 6000), True)],
                         ids=["1", "4", "12", "13000_candidates"])
def test_soft_merge_equals_oracle(n_tiles, hw, full):
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    from test_large_image_gpu import _records
    P, M = 512, 100
    org = slice_origins(hw, P, 0.25)[:n_tiles]
    recs = _records(n_tiles, P, M, seed=n_tiles, full=full)
    origins = [org[i:i + 4] for i in range(0, n_tiles, 4)]
    got = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25, nms_type="soft_nms")
    tiles, offs, src = [], [], []
    for r, (rec, o) in enumerate(zip(recs, origins)):
        host = rec.to_host(non_blocking=False)
        for b, xy in enumerate(o):
            n = int(host.counts[b])
            rows = host.rows[b, :n]
            tiles.append(dict(bboxes=rows[:, :4], scores=rows[:, 4], labels=rows[:, 5].long()))
            offs.append(xy)
            src += [(r, b, s) for s in range(n)]
    ref, keep = R.merge_results_by_nms(tiles, offs, hw, dict(type="soft_nms", iou_threshold=0.25), patch=P)
    assert (keep.numel() >= R.SPLIT_THR) == full
    assert got["bboxes"].shape[0] == keep.numel() > 0
    assert torch.equal(got["bboxes"].cpu(), ref["bboxes"])
    assert torch.equal(got["scores"].cpu(), ref["scores"])
    assert torch.equal(got["labels"].cpu(), ref["labels"])
    assert torch.equal(got["source"], torch.tensor(src, dtype=torch.int64).view(-1, 3)[keep])
    hard = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25)
    assert got["bboxes"].shape[0] >= hard["bboxes"].shape[0]
    # score_thr filters the merged rows
    cut = merge_tile_records(recs, origins, hw, merge_iou_thr=0.25, nms_type="soft_nms", score_thr=0.5)
    k = got["scores"] >= 0.5
    assert torch.equal(cut["scores"], got["scores"][k]) and torch.equal(cut["source"], got["source"][k.cpu()])


def test_predict_large_image_soft_merge_and_cli(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from rsprompter_b200.large_image import coco_results, main, predict_large_image, run_tiles
    from rsprompter_b200.results import mask_to_coco_rle
    from test_large_image_gpu import _model, _model_cfg, _scene
    from oracle import restate_large_image as oracle
    model = _model("query")
    scene = _scene(700, 900, seed=12)
    ds = predict_large_image(model, scene, merge_nms_type="soft_nms")
    records, batches = run_tiles(model, scene)
    tiles, offs = [], []
    for rec, org in zip(records, batches):
        inst = rec.to_host(non_blocking=False).instances()
        tiles += inst[:len(org)]
        offs += org
    P = model.backbone.vision_encoder.arch.image_size
    boxes_only = [{k: t[k] for k in ("bboxes", "scores", "labels")} for t in tiles]
    ref, keep = R.merge_results_by_nms(boxes_only, offs, (700, 900), dict(type="soft_nms", iou_threshold=0.25),
                                       patch=P)
    p = ds.pred_instances
    assert len(p.masks) == keep.numel() > 0
    assert torch.equal(p.bboxes.cpu(), ref["bboxes"]) and torch.equal(p.scores.cpu(), ref["scores"])
    masks = [m for t in tiles for m in t["masks"]]
    tile_of = [i for i, t in enumerate(tiles) for _ in range(t["masks"].shape[0])]
    rles = [mask_to_coco_rle(oracle.shift_masks(masks[k][None], offs[tile_of[k]], (700, 900))[0])["counts"]
            for k in keep.tolist()]
    assert [m["counts"] for m in p.masks] == rles
    # the CLI
    cfg = tmp_path / "cfg.py"
    cfg.write_text("model = " + repr(_model_cfg("query")) + "\n")
    ckpt = tmp_path / "model.pth"
    torch.save(dict(state_dict=model.state_dict()), ckpt)
    img = tmp_path / "scene.png"
    cv2.imwrite(str(img), scene)
    out = tmp_path / "results.json"
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(out), "--merge-nms-type", "soft_nms"])
    assert json.loads(out.read_text()) == json.loads(json.dumps(coco_results(ds)))
