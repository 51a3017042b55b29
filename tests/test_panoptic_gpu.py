"""Panoptic output of the query detectors on the GPU against oracle/restate_panoptic.py run on CUDA tensors: the kernels
byte for byte where the resize is the identity (the fixture's adversarial cases, nq 100 and 300), the resampled paths
on blob logits whose near-tie band is empty, both detectors end to end, and the flag defaults."""
import os

import pytest
import torch

from oracle import restate_panoptic as rp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FX = torch.load(os.path.join(ROOT, "tests", "golden", "reference_panoptic.pt"), weights_only=False)
EPS = 2.0 ** -20


def _head(num_things, num_classes, cfg):
    from rsprompter_b200.registry import MODELS
    return MODELS.build(dict(type="RSMaskFormerFusionHead", num_things_classes=num_things,
                             num_stuff_classes=num_classes - num_things, test_cfg=dict(cfg)))


def _check_stats(got: dict, st: dict):
    q = torch.tensor(st["query"], dtype=torch.long)
    for k in ("mask_area", "original_area", "segment_id"):
        assert got[k].cpu()[q].tolist() == st[k], k
    notkept = torch.ones(got["mask_area"].numel(), dtype=torch.bool)
    notkept[q] = False
    assert (got["segment_id"].cpu()[notkept] == -1).all() and (got["mask_area"].cpu()[notkept] == 0).all()


@pytest.mark.parametrize("name", sorted(FX["cases"]))
def test_kernels_byte_exact_on_the_fixture(name):
    cfg = FX["cases"][name]["test_cfg"]
    C, T = FX["num_classes"], FX["num_things_classes"]
    cls, mp = FX["mask_cls"].cuda(), FX["mask_pred"].cuda()
    pans, stats = _head(T, C, cfg).panoptic_postprocess_batched(cls[None], mp, tuple(mp.shape[-2:]))
    ref, st = rp.panoptic_postprocess(cls, mp, C, T, cfg, stats=True)
    assert pans[0].dtype == torch.int32 and torch.equal(pans[0], ref)
    assert torch.equal(pans[0].cpu(), FX["cases"][name]["pan"])
    _check_stats(stats[0], st)


def _blobs(n, hm, wm, g, steep=1.7, floor=None):
    yy, xx = torch.meshgrid(torch.arange(hm, dtype=torch.float32), torch.arange(wm, dtype=torch.float32), indexing="ij")
    cy, cx = torch.rand(n, 1, 1, generator=g) * hm, torch.rand(n, 1, 1, generator=g) * wm
    r = 1.5 + torch.rand(n, 1, 1, generator=g) * hm / 6
    v = (r - ((yy - cy) ** 2 + (xx - cx) ** 2).sqrt()) * steep
    return v if floor is None else v.clamp(min=floor)


@pytest.mark.parametrize("nq", [100, 300])
@pytest.mark.parametrize("flt", [False, True])
def test_kernels_byte_exact_at_output_size(nq, flt):
    """Identity resize: the map and both area vectors equal the oracle's exactly.  Duplicated queries make exact ties,
    exact-zero and -1e-8 logits make sigmoid exactly 0.5, stuff classes merge, and some images keep nothing."""
    g = torch.Generator().manual_seed(nq)
    B, H, W, C, T = 3, 96, 80, 9, 6
    cls = torch.randn(B, nq, C + 1, generator=g)
    cls[:, :, :C] += 4.0 * (torch.rand(B, nq, C, generator=g) > 0.8)
    mp = _blobs(B * nq, H, W, g, steep=0.9).view(B, nq, H, W)
    mp[:, 1::7] = mp[:, 0::7][:, :mp[:, 1::7].shape[1]]               # exact ties ...
    cls[:, 1::7] = cls[:, 0::7][:, :cls[:, 1::7].shape[1]]            # ... with the same scores
    mp[:, :, 10:12, :] = 0.0
    mp[:, :, 20:21, :] = -1e-8
    cls[2] = -5.0
    cls[2, :, C] = 5.0                                                 # image 2: every query on the no-object class
    cfg = dict(object_mask_thr=0.5, iou_thr=0.6, filter_low_score=flt)
    cls, mp = cls.cuda(), mp.cuda()
    pans, stats = _head(T, C, cfg).panoptic_postprocess_batched(cls, mp.view(B * nq, H, W).contiguous(), (H, W))
    kept = 0
    for b in range(B):
        ref, st = rp.panoptic_postprocess(cls[b], mp[b], C, T, cfg, stats=True)
        assert torch.equal(pans[b], ref), b
        _check_stats(stats[b], st)
        kept += len(st["query"])
    assert kept > 20 and (pans[2] == C).all()


def _band_ok(cls, up, cfg, C):
    """No pixel whose top-two prob gap, or any kept query's |sigmoid - 0.5|, is below 2^-20."""
    scores, labels = torch.softmax(cls, -1).max(-1)
    keep = labels.ne(C) & (scores > cfg.get("object_mask_thr", 0.8))
    if keep.sum() < 2:
        return False
    sig = up[keep].sigmoid()
    prob = scores[keep].view(-1, 1, 1) * sig
    top = prob.topk(2, dim=0).values
    return bool(((top[0] - top[1]) >= EPS).all() and ((sig - 0.5).abs() >= EPS).all())


def _resampled_case(seed, B, nq, hm, C):
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(B, nq, C + 1, generator=g)
    cls[:, :, :C] += 3.0 * (torch.rand(B, nq, C, generator=g) > 0.85)
    logits = _blobs(B * nq, hm, hm, g, steep=40.0, floor=-30.0)
    logits[::nq] = -2.0                                                 # one background query per image
    cls[:, 0, :C] = 0.0
    cls[:, 0, 0] = 6.0
    return cls.cuda(), logits.cuda().contiguous()


@pytest.mark.parametrize("path", ["x4", "rescale", "no_rescale"])
def test_resampled_paths_match_oracle(path):
    B, nq, hm, C, T = 2, 100, 32, 6, 4
    batch, ori = (4 * hm, 4 * hm), (150, 110)
    s = min(batch[0] / ori[0], batch[1] / ori[1])
    new = (int(ori[0] * s + 0.5), int(ori[1] * s + 0.5))
    sf = (new[1] / ori[1], new[0] / ori[0])
    meta = dict(ori_shape=ori, scale_factor=sf)
    m = dict(ori_hw=ori, crop_hw=(min(int(ori[0] * sf[1]), batch[0]), min(int(ori[1] * sf[0]), batch[1])), scale_factor=sf)
    cfg = dict(object_mask_thr=0.4, iou_thr=0.5)
    for seed in range(20):       # seeded inputs whose oracle masks have no pixel in the near-tie band
        cls, logits = _resampled_case(seed, B, nq, hm, C)
        ups = []
        for b in range(B):
            lg = logits[b * nq:(b + 1) * nq]
            ups.append(rp.resample(lg, batch) if path == "x4" else rp.resample(lg, batch, meta, rescale=path == "rescale"))
        if all(_band_ok(cls[b], ups[b], cfg, C) for b in range(B)):
            break
    assert all(_band_ok(cls[b], ups[b], cfg, C) for b in range(B))
    metas = None if path == "x4" else [m] * B
    pans, stats = _head(T, C, cfg).panoptic_postprocess_batched(cls, logits, batch, metas=metas,
                                                                 rescale=path == "rescale")
    for b in range(B):
        ref, st = rp.panoptic_postprocess(cls[b], ups[b], C, T, cfg, stats=True)
        assert pans[b].shape == ref.shape and torch.equal(pans[b], ref)
        _check_stats(stats[b], st)
        assert sum(1 for sid in st["segment_id"] if sid >= 0) >= 2


# ------------------------------------------------------------------------------ end to end
NCLS = 10


def _model(kind):
    from rsprompter_b200 import model_configs, sam_config, synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    from rsprompter_b200.registry import MODELS
    arch = sam_config.VISION_ARCHS["base"]
    sel = SELECT_LAYERS["base"]
    if kind == "query":
        m = MODELS.build(model_configs.query_model_cfg("base", NCLS, prompt_shape=(100, 5)))
        sd = synthetic.query_detector_state_dict(arch, NCLS, len(sel), nq=100, seed=3)
    else:
        m = MODELS.build(model_configs.mask2former_model_cfg("base", NCLS, num_queries=100))
        sd = synthetic.mask2former_detector_state_dict(arch, NCLS, len(sel), nq=100, seed=6)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _set_cfg(m, **cfg):
    from rsprompter_b200.registry import ConfigDict
    c = ConfigDict(cfg)
    m.test_cfg = c
    m.panoptic_fusion_head.test_cfg = c


def _samples(resized):
    from rsprompter_b200.registry import make_data_samples
    ds = make_data_samples(2, 1024)
    if resized:                    # NWPU-like: 800 x 1000 and 700 x 933 images resized to a 1024 long side, padded
        ds[0].set_metainfo(dict(ori_shape=(800, 1000), img_shape=(819, 1024), scale_factor=(1.024, 1.02375)))
        ds[1].set_metainfo(dict(ori_shape=(700, 933), img_shape=(768, 1024), scale_factor=(1024 / 933, 768 / 700)))
    return ds


@pytest.mark.parametrize("kind", ["query", "mask2former"])
def test_detectors_end_to_end(kind):
    m = _model(kind)
    torch.manual_seed(11)
    x = torch.randn(2, 3, 1024, 1024).cuda()
    thr = 0.0
    raw = m.predict_raw(x)
    cls, logits = raw["cls"].clone(), raw["mask_logits"].clone()
    nq = cls.shape[1]
    for resized in (False, True):
        cfg = dict(object_mask_thr=thr, iou_thr=0.8, max_per_image=100)
        _set_cfg(m, panoptic_on=False, instance_on=True, **cfg)
        inst_only = m.predict(x, _samples(resized))
        _set_cfg(m, panoptic_on=True, instance_on=True, **cfg)
        both = m.predict(x, _samples(resized))
        hw, metas = m._metas(_samples(resized), x)
        for b in range(2):
            a, c = inst_only[b].pred_instances, both[b].pred_instances
            for k in ("bboxes", "scores", "labels", "masks"):
                assert torch.equal(getattr(a, k), getattr(c, k)), k
            lg = logits[b * nq:(b + 1) * nq]
            meta = None if metas[b] is None else dict(ori_shape=metas[b]["ori_hw"],
                                                      scale_factor=metas[b]["scale_factor"])
            up = rp.resample(lg, hw, meta)
            fh = m.panoptic_fusion_head
            ref, st = rp.panoptic_postprocess(cls[b], up, fh.num_classes, fh.num_things_classes, cfg, stats=True)
            pan = both[b].pred_panoptic_seg.sem_seg
            assert pan.shape == ref.shape and pan.dtype == torch.int32
            scores, labels = torch.softmax(cls[b], -1).max(-1)
            keep = labels.ne(fh.num_classes) & (scores > thr)
            assert keep.sum() > 0
            if _band_ok(cls[b], up, cfg, fh.num_classes):
                assert torch.equal(pan, ref)
            else:              # near-tie pixels may go either way; every other pixel must agree
                sig = up[keep].sigmoid()
                prob = scores[keep].view(-1, 1, 1) * sig
                top = prob.topk(min(2, int(keep.sum())), dim=0).values
                band = ((sig - 0.5).abs() < EPS).any(0)
                if top.shape[0] > 1:
                    band |= (top[0] - top[1]) < EPS
                assert ((pan[0] != ref[0]) & ~band).sum().item() == 0
    # the post-processing itself makes no host synchronisation
    _set_cfg(m, object_mask_thr=thr)
    hw, metas = m._metas(_samples(True), x)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.panoptic_fusion_head.panoptic_postprocess_batched(cls, logits, hw, metas=metas)
        m.panoptic_fusion_head.panoptic_postprocess_batched(cls, logits, hw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_panoptic_on_missing_gives_panoptic_only():
    m = _model("query")
    _set_cfg(m, max_per_image=100)          # no panoptic_on / instance_on: the reference's defaults
    torch.manual_seed(5)
    out = m.predict(torch.randn(1, 3, 1024, 1024).cuda())
    assert "pred_instances" not in out[0]
    pan = out[0].pred_panoptic_seg.sem_seg
    assert pan.shape == (1, 1024, 1024) and pan.dtype == torch.int32 and pan.is_cuda
