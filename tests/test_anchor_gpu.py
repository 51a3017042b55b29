"""RSPrompter-anchor head path on the GPU vs the CPU oracle, stage by stage.  Continuous stages are
compared with a bf16 tolerance on the same inputs; index-producing stages (top-k / decode / NMS /
compaction) are checked EXACTLY by running the oracle's post-processing on the tensors the GPU
stage produced."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NUM_CLASSES = 10


def _relerr(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item() / max(b.abs().max().item(), 1e-6)


@pytest.fixture(scope="module")
def model_and_sd():
    from rsprompter_b200 import model_configs, synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS
    cfg = model_configs.anchor_model_cfg("base", NUM_CLASSES)
    m = MODELS.build(cfg)
    sd = synthetic.anchor_detector_state_dict(VISION_ARCHS["base"], NUM_CLASSES, 6, seed=3)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def _assert_same_detections(boxes, scores, ref_boxes, ref_scores, labels=None, ref_labels=None):
    """Same detections after a canonical sort: the reference's own order among (near-)equal scores is
    unspecified (unstable sort, rpn_head.py:208) and device sigmoid/softmax differ from the CPU by an
    ulp, so rows are matched by content: every reference row must have an identical row here."""
    assert boxes.shape == ref_boxes.shape
    a = torch.cat([boxes, scores[:, None]], 1)
    b = torch.cat([ref_boxes, ref_scores[:, None]], 1)
    if labels is not None:
        a = torch.cat([a, labels[:, None].float()], 1)
        b = torch.cat([b, ref_labels[:, None].float()], 1)
    d = (a[:, None, :] - b[None, :, :]).abs()
    d[..., 4] *= 100.0          # scores: 2e-5 tolerance vs 2e-3 on coordinates
    d = d.amax(dim=2)
    assert d.min(dim=1).values.max().item() < 2e-3, "a detection here has no match in the oracle's list"
    assert d.min(dim=0).values.max().item() < 2e-3, "an oracle detection is missing here"
    # and the order agrees wherever scores are separated by more than the ulp-level tolerance
    assert (scores[:-1] >= scores[1:] - 1e-6).all()


def _sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def _nhwc_bf16(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()


def test_neck_matches_oracle(model_and_sd):
    from oracle import restate_anchor as ra
    m, sd = model_and_sd
    g = torch.Generator().manual_seed(5)
    hidden = [torch.randn(1, 64, 64, 768, generator=g) for _ in range(13)]
    agg_sd, fpn_sd = _sub(sd, "neck.feature_aggregator."), _sub(sd, "neck.feature_spliter.")
    ref_agg = ra.feature_aggregator(agg_sd, hidden, list(range(1, 13, 2)))
    ref = ra.simple_fpn(fpn_sd, ref_agg)
    agg = m.neck.feature_aggregator.forward_nhwc([h.cuda() for h in hidden])
    assert _relerr(agg.permute(0, 3, 1, 2), ref_agg) < 3e-2
    outs = m.neck.forward_nhwc([h.cuda() for h in hidden])
    torch.cuda.synchronize()
    assert len(outs) == 5
    for o, r in zip(outs, ref):
        assert tuple(o.shape) == (r.shape[0], r.shape[2], r.shape[3], r.shape[1])
        assert _relerr(o.permute(0, 3, 1, 2), r) < 4e-2


def test_rpn_head_and_proposals(model_and_sd):
    from oracle import restate_anchor as ra
    m, sd = model_and_sd
    g = torch.Generator().manual_seed(6)
    B = 2
    sizes = [256, 128, 64, 32, 16]
    feats = [torch.randn(B, 256, s, s, generator=g).to(torch.bfloat16).float() for s in sizes]
    cap = {}
    props, scores, cnt = m.rpn_head.predict_nhwc([_nhwc_bf16(f) for f in feats], (1024, 1024), capture=cap)
    torch.cuda.synchronize()
    ref = ra.rpn_forward(_sub(sd, "rpn_head."), feats, prefix="")
    strides = [4, 8, 16, 32, 64]
    A = 6
    for lvl, (c_ref, r_ref) in enumerate(ref):
        out = cap["head_out"][lvl].cpu()
        assert _relerr(out[..., :A].permute(0, 3, 1, 2), c_ref) < 2e-2
        assert _relerr(out[..., A:5 * A].permute(0, 3, 1, 2), r_ref) < 2e-2
    # exact post-processing on the GPU head outputs
    for b in range(B):
        cls_l, reg_l, pri_l = [], [], []
        for lvl, s in enumerate(sizes):
            out = cap["head_out"][lvl][b].cpu()
            cls_l.append(out[..., :A].permute(2, 0, 1))
            reg_l.append(out[..., A:5 * A].permute(2, 0, 1))
            pri_l.append(ra.grid_anchors((s, s), strides[lvl], ra.base_anchors(strides[lvl], [4, 8], [0.5, 1.0, 2.0])))
        pb, ps = ra.rpn_predict_single(cls_l, reg_l, pri_l, (1024, 1024))
        n = cnt[b].item()
        assert n == pb.shape[0], f"proposal count {n} vs oracle {pb.shape[0]}"
        _assert_same_detections(props[b, :n].cpu(), scores[b, :n].cpu(), pb, ps)
        assert (props[b, n:] == 0).all()


def test_roi_head_stages(model_and_sd):
    from oracle import restate_anchor as ra
    m, sd = model_and_sd
    g = torch.Generator().manual_seed(7)
    B, K = 2, 200
    sizes = [256, 128, 64, 32, 16]
    feats = [torch.randn(B, 256, s, s, generator=g).to(torch.bfloat16).float() for s in sizes]
    # plausible proposals: random boxes of assorted sizes
    ctr = torch.rand(B, K, 2, generator=g) * 1024
    wh = torch.exp(torch.rand(B, K, 2, generator=g) * 5.0 + 1.5)
    props = torch.cat([(ctr - wh / 2).clamp(0, 1024), (ctr + wh / 2).clamp(0, 1024)], dim=2)
    pcnt = torch.tensor([K, K - 37], dtype=torch.int32)
    props[1, K - 37:] = 0
    emb_rows = torch.randn(B * 4096, 256, generator=g).cuda()
    pos_rows = torch.randn(4096, 256, generator=g).cuda()
    cap = {}
    r = m.roi_head.predict_nhwc([_nhwc_bf16(f) for f in feats], props.cuda(), pcnt.cuda(), (1024, 1024),
                                emb_rows, pos_rows, (64, 64), capture=cap)
    torch.cuda.synchronize()
    # RoIAlign(7x7) with the extra PE + bbox FCs vs oracle
    feats_pe = ra.add_extra_pe(feats)
    rois = cap["rois"].cpu()
    ref7 = ra.roi_extract(feats_pe[:4], rois, 7)
    got7 = cap["roi_feats7"].float().cpu().view(-1, 7, 7, 256).permute(0, 3, 1, 2)
    assert _relerr(got7, ref7) < 2e-2
    bsd = _sub(sd, "roi_head.bbox_head.")
    cls_ref, reg_ref = ra.bbox_head_forward(bsd, ref7, prefix="")
    assert _relerr(cap["cls"], cls_ref) < 3e-2 and _relerr(cap["reg"], reg_ref) < 3e-2
    # exact detection post-processing on the GPU logits
    for b in range(B):
        n_roi = pcnt[b].item()
        sl = slice(b * K, b * K + n_roi)
        db, ds, dl = ra.bbox_predict_single(rois[sl], cap["cls"][sl].cpu(), cap["reg"][sl].cpu(), (1024, 1024),
                                            NUM_CLASSES)
        n = r["counts"][b].item()
        assert n == db.shape[0]
        _assert_same_detections(r["bboxes"][b, :n].cpu(), r["scores"][b, :n].cpu(), db, ds,
                                r["labels"][b, :n].cpu(), dl)
    # mask branch: RoIAlign(14x14) + prompt generator
    mrois = cap["mask_rois"].cpu()
    ref14 = ra.roi_extract(feats_pe[:4], mrois, 14)
    got14 = cap["roi_feats14"].float().cpu().view(-1, 14, 14, 256).permute(0, 3, 1, 2)
    assert _relerr(got14, ref14) < 2e-2
    sparse_ref = ra.mask_head_prompts(_sub(sd, "roi_head.mask_head."), ref14, 5, prefix="")
    sparse = m.roi_head.mask_head.prompts_from_roi_feats(cap["roi_feats14"])
    assert sparse.shape == sparse_ref.shape == (B * 100, 5, 256)
    assert _relerr(sparse, sparse_ref) < 3e-2
    assert r["mask_logits"].shape == (B * 100, 1, 256, 256)


@pytest.mark.parametrize("hm,size", [(256, (1024, 1024)), (64, (256, 256)), (256, (768, 768)), (48, (176, 208))])
def test_mask_paste_to_size_matches_oracle(hm, size):
    """x4 tiles (the shipped case: logits are image / 4) and the generic-scale kernel, borders included."""
    from oracle import restate_anchor as ra
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(8)
    logits = torch.randn(5, 1, hm, hm, generator=g) * 3
    ref = ra.mask_postprocess(logits, size, 0.5)
    got = _lib.mask_paste(logits[:, 0].contiguous().cuda(), 0.5, raw=False, size=size)
    torch.cuda.synchronize()
    assert got.dtype == torch.bool and got.shape == ref.shape
    assert (got.cpu() != ref).float().mean().item() < 1e-5
    assert torch.equal(got.cpu()[:, :2], ref[:, :2]) or (got.cpu()[:, :2] != ref[:, :2]).float().mean().item() < 1e-4


def test_end_to_end_predict_contract(model_and_sd):
    m, _ = model_and_sd
    from rsprompter_b200.registry import make_data_samples
    torch.manual_seed(0)
    x = torch.randn(2, 3, 1024, 1024, device="cuda")
    out = m.predict(x, make_data_samples(2, 1024))
    assert len(out) == 2
    for ds in out:
        p = ds.pred_instances
        n = len(p)
        assert 0 <= n <= 100
        assert p.bboxes.shape == (n, 4) and p.scores.shape == (n,) and p.labels.shape == (n,)
        assert p.masks.shape == (n, 1024, 1024) and p.masks.dtype == torch.bool
        assert p.labels.dtype == torch.int64 and (p.labels >= 0).all() and (p.labels < NUM_CLASSES).all()
        assert (p.scores[:-1] >= p.scores[1:]).all()
    out2 = m.predict(x, make_data_samples(2, 1024))
    assert torch.equal(out[0].pred_instances.bboxes, out2[0].pred_instances.bboxes)


@pytest.mark.parametrize("ori,batch", [((120, 200), (256, 256)), ((512, 512), (1024, 1024)), ((300, 180), (256, 256))])
def test_mask_paste_with_rescale_matches_oracle(ori, batch):
    """Resized + padded images (M:1763-1777): sigmoid -> batch shape -> crop -> ori_shape -> threshold, no intermediate."""
    from oracle import restate_anchor as ra
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(9)
    hm = batch[0] // 4
    s = min(batch[0] / ori[0], batch[1] / ori[1])
    new_hw = (int(ori[0] * s + 0.5), int(ori[1] * s + 0.5))
    meta = dict(ori_shape=ori, batch_input_shape=batch, scale_factor=(new_hw[1] / ori[1], new_hw[0] / ori[0]))
    logits = torch.randn(4, 1, hm, hm, generator=g) * 3
    boxes = torch.rand(4, 4, generator=g) * 200
    ref, ref_boxes = ra.mask_postprocess_rescale(logits, boxes.clone(), meta, 0.5)
    sf = meta["scale_factor"]
    crop = (min(int(ori[0] * sf[1]), batch[0]), min(int(ori[1] * sf[0]), batch[1]))
    got = _lib.mask_paste(logits[:, 0].contiguous().cuda(), 0.5, raw=False, rescale=(batch, crop, ori))
    torch.cuda.synchronize()
    assert got.shape == ref.shape and got.dtype == torch.bool
    assert (got.cpu() != ref).float().mean().item() < 2e-5


def test_predict_rescales_to_original_image(model_and_sd):
    """predict() with the metainfo of a keep-ratio resized, padded image: boxes / scale_factor, masks at ori_shape."""
    from rsprompter_b200.registry import make_data_samples
    m, _ = model_and_sd
    torch.manual_seed(5)
    x = torch.randn(2, 3, 1024, 1024).cuda()
    base_samples = make_data_samples(2, (1024, 1024))
    base_samples[1].set_metainfo(dict(img_shape=(768, 1024)))              # same per-image clip, no rescale
    base = m.predict(x, base_samples)
    samples = make_data_samples(2, (1024, 1024))
    samples[1].set_metainfo(dict(ori_shape=(600, 800), img_shape=(768, 1024), scale_factor=(1.28, 1.28),
                                 batch_input_shape=(1024, 1024)))
    out = m.predict(x, samples)
    torch.cuda.synchronize()
    p0, p1, b1 = out[0].pred_instances, out[1].pred_instances, base[1].pred_instances
    assert torch.equal(p0.masks, base[0].pred_instances.masks)            # untouched image: same fast-path result
    n = p1.scores.numel()
    assert p1.masks.shape == (n, 600, 800) and torch.equal(p1.scores, b1.scores)
    assert torch.allclose(p1.bboxes, b1.bboxes / 1.28, rtol=1e-6, atol=1e-4)


def test_cuda_graph_replay_equals_eager(model_and_sd):
    """enable_cuda_graphs(): the captured forward replays to the same detections as the eager launch sequence."""
    m, _ = model_and_sd
    torch.manual_seed(11)
    xs = [torch.randn(2, 3, 1024, 1024).cuda() for _ in range(2)]
    eager = [m.predict(x) for x in xs]
    eager = [[(d.pred_instances.bboxes.clone(), d.pred_instances.scores.clone(), d.pred_instances.masks.clone())
              for d in out] for out in eager]
    m.enable_cuda_graphs()
    try:
        for rep in range(2):
            for x, ref in zip(xs, eager):
                out = m.predict(x)
                for d, (b, s, k) in zip(out, ref):
                    assert torch.equal(d.pred_instances.bboxes, b) and torch.equal(d.pred_instances.scores, s)
                    assert torch.equal(d.pred_instances.masks, k)
    finally:
        m.enable_cuda_graphs(False)


def test_per_image_img_shape_clipping(model_and_sd):
    """Batches whose images were padded to a common shape: the RPN (rpn_head.py:208-215) and the bbox head
    (bbox_head.py:545-548) clip every image's boxes to its own img_meta['img_shape'], carried as a device [B, 2]
    tensor; exact against the oracle's post-processing of the same logits with the per-image shapes."""
    from oracle import restate_anchor as ra
    m, sd = model_and_sd
    g = torch.Generator().manual_seed(16)
    B, K = 2, 150
    shapes = [(1024, 1024), (800, 904)]
    sh = torch.tensor(shapes, dtype=torch.float32).cuda()
    sizes = [256, 128, 64, 32, 16]
    feats = [torch.randn(B, 256, s, s, generator=g).to(torch.bfloat16).float() for s in sizes]
    nh = [_nhwc_bf16(f) for f in feats]
    cap = {}
    props, scores, cnt = m.rpn_head.predict_nhwc(nh, (1024, 1024), capture=cap, img_shapes=sh)
    strides, A = [4, 8, 16, 32, 64], 6
    for b in range(B):
        cls_l, reg_l, pri_l = [], [], []
        for lvl, s in enumerate(sizes):
            out = cap["head_out"][lvl][b].cpu()
            cls_l.append(out[..., :A].permute(2, 0, 1))
            reg_l.append(out[..., A:5 * A].permute(2, 0, 1))
            pri_l.append(ra.grid_anchors((s, s), strides[lvl], ra.base_anchors(strides[lvl], [4, 8], [0.5, 1.0, 2.0])))
        pb, ps = ra.rpn_predict_single(cls_l, reg_l, pri_l, shapes[b])
        n = cnt[b].item()
        assert n == pb.shape[0]
        _assert_same_detections(props[b, :n].cpu(), scores[b, :n].cpu(), pb, ps)
        assert props[b, :n, 0::2].max().item() <= shapes[b][1] and props[b, :n, 1::2].max().item() <= shapes[b][0]
    assert props[1, :, 0::2].max().item() > 890            # the clip is the image's, not a tighter one
    # bbox head on random proposals
    ctr = torch.rand(B, K, 2, generator=g) * 1024
    wh = torch.exp(torch.rand(B, K, 2, generator=g) * 5.0 + 1.5)
    rp = torch.cat([(ctr - wh / 2).clamp(0, 1024), (ctr + wh / 2).clamp(0, 1024)], dim=2)
    pcnt = torch.tensor([K, K], dtype=torch.int32)
    emb_rows = torch.randn(B * 4096, 256, generator=g).cuda()
    pos_rows = torch.randn(4096, 256, generator=g).cuda()
    cap = {}
    r = m.roi_head.predict_nhwc(nh, rp.cuda(), pcnt.cuda(), (1024, 1024), emb_rows, pos_rows, (64, 64), capture=cap,
                                img_shapes=sh)
    torch.cuda.synchronize()
    rois = cap["rois"].cpu()
    for b in range(B):
        sl = slice(b * K, (b + 1) * K)
        db, ds, dl = ra.bbox_predict_single(rois[sl], cap["cls"][sl].cpu(), cap["reg"][sl].cpu(), shapes[b], NUM_CLASSES)
        n = r["counts"][b].item()
        assert n == db.shape[0]
        _assert_same_detections(r["bboxes"][b, :n].cpu(), r["scores"][b, :n].cpu(), db, ds, r["labels"][b, :n].cpu(), dl)
        assert r["bboxes"][b, :n, 0::2].max().item() <= shapes[b][1] and r["bboxes"][b, :n, 1::2].max().item() <= shapes[b][0]


def test_predict_attaches_per_image_shapes(model_and_sd):
    """predict() with data samples whose img_shape is smaller than the batch shape: detections stay inside the image
    (eager and graph mode); an image whose img_shape equals the batch shape is unaffected."""
    from rsprompter_b200.registry import make_data_samples
    m, _ = model_and_sd
    torch.manual_seed(17)
    x = torch.randn(2, 3, 1024, 1024).cuda()
    base = m.predict(x, make_data_samples(2, 1024))
    ds = make_data_samples(2, 1024)
    ds[1].set_metainfo(dict(img_shape=(640, 768)))
    out = m.predict(x, ds)
    p0, p1 = out[0].pred_instances, out[1].pred_instances
    assert torch.equal(p0.bboxes, base[0].pred_instances.bboxes) and torch.equal(p0.masks, base[0].pred_instances.masks)
    assert len(p1) > 0 and p1.bboxes[:, 0::2].max().item() <= 768 and p1.bboxes[:, 1::2].max().item() <= 640
    assert base[1].pred_instances.bboxes[:, 0::2].max().item() > 768        # the un-clipped run does reach the padding
    m.enable_cuda_graphs()
    try:
        ds2 = make_data_samples(2, 1024)
        ds2[1].set_metainfo(dict(img_shape=(640, 768)))
        g1 = m.predict(x, ds2)
        ds3 = make_data_samples(2, 1024)
        ds3[1].set_metainfo(dict(img_shape=(512, 1000)))                      # same graph, refreshed shape buffer
        g2 = m.predict(x, ds3)
        torch.cuda.synchronize()
        assert torch.equal(g1[1].pred_instances.bboxes, p1.bboxes) and torch.equal(g1[1].pred_instances.scores, p1.scores)
        b2 = g2[1].pred_instances.bboxes
        assert b2[:, 1::2].max().item() <= 512 and b2[:, 0::2].max().item() <= 1000 and b2[:, 0::2].max().item() > 768
    finally:
        m.enable_cuda_graphs(False)


@pytest.mark.parametrize("n,K", [(3000, 50), (700, 1000), (64, 1)])
def test_nms_early_stop_keeps_the_same_first_k(n, K):
    """rsp_nms_batched with max_keep > 0: stopping the greedy scan after max_keep kept candidates leaves the first K kept
    ones (all a caller of batched_nms(...)[:max_per_img] reads) unchanged."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(n + K)
    B = 3
    ctr = torch.rand(B, n, 2, generator=g) * 600
    wh = torch.rand(B, n, 2, generator=g) * 120 + 4
    boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], dim=2).cuda().contiguous()
    scores = torch.sort(torch.rand(B, n, generator=g), dim=1, descending=True).values.cuda().contiguous()
    ids = torch.randint(0, 4, (B, n), generator=g).cuda()
    nvalid = torch.tensor([n, n - 17, max(n // 2, 1)], dtype=torch.int32).cuda()
    full = _lib.nms_batched(boxes, ids, nvalid, 0.5)
    part = _lib.nms_batched(boxes, ids, nvalid, 0.5, max_keep=K)
    a = _lib.compact_keep(full, boxes, scores, ids, K)
    b = _lib.compact_keep(part, boxes, scores, ids, K)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert (part <= full).all()
