"""COCO RLE of predicted masks on the device (rsp_mask_rle_*, results.encode_mask_results, test_cfg.rle_masks): the
strings must be byte for byte those of results.mask_to_coco_rle (pycocotools' rleEncode + rleToString), from bool /
uint8 masks and from the bit-packed record payload, and the detectors' rle_masks output must decode to the masks they
return without it."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NUM_CLASSES = 10


def _blobs(n, h, w, seed):
    """n masks of a few filled ellipses each (object-shaped: long runs, few transitions per column)."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = np.zeros((n, h, w), dtype=bool)
    for i in range(n):
        for _ in range(3):
            cy, cx = g.uniform(0, h), g.uniform(0, w)
            ry, rx = g.uniform(1, max(2, h / 3)), g.uniform(1, max(2, w / 3))
            out[i] |= ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
    return out


def _single(h, w, idx):
    m = np.zeros((1, h, w), dtype=bool)
    m.reshape(-1)[idx] = True
    return m


_G = np.random.default_rng(0)
_YY, _XX = np.mgrid[0:512, 0:512]
CASES = {
    "zeros": lambda: np.zeros((1, 37, 53), dtype=bool),
    "ones": lambda: np.ones((1, 37, 53), dtype=bool),
    "first_pixel": lambda: _single(37, 53, 0),
    "last_pixel": lambda: _single(37, 53, -1),
    "h1": lambda: _G.random((2, 1, 300)) < 0.3,
    "w1": lambda: _G.random((2, 300, 1)) < 0.3,
    "checkerboard": lambda: ((_YY + _XX) % 2 == 1)[None],                     # a run per pixel
    "row_stripes": lambda: (_YY % 4 < 2)[None, :, :300],                      # runs cross column boundaries
    "col_stripes": lambda: (_XX % 6 < 3)[None, :300],
    "noise_1024": lambda: _G.random((1, 1024, 1024)) < 0.5,                   # multi-char and negative differences
    "zeros_2048": lambda: np.zeros((1, 2048, 2048), dtype=bool),             # a count >= 2^20
    "blobs_800x1333": lambda: _blobs(2, 800, 1333, 1),
    "blobs_4097x3": lambda: _blobs(2, 4097, 3, 2),
    "blobs_3x4097": lambda: _blobs(2, 3, 4097, 3),
    "blobs_w_not_multiple_of_8": lambda: _blobs(3, 61, 131, 4),
}


def _ref(masks):
    from rsprompter_b200.results import mask_to_coco_rle
    return [mask_to_coco_rle(m) for m in masks]


@pytest.mark.parametrize("name", list(CASES))
def test_encode_equals_host_rle_bool_and_bits(name):
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import encode_mask_results
    m = CASES[name]()
    ref = _ref(m)
    dev = torch.from_numpy(m).cuda()
    assert encode_mask_results(dev) == ref
    assert encode_mask_results(dev.to(torch.uint8) * 7) == ref          # any nonzero byte is set
    bits = _lib.pack_mask_bits(dev)
    assert _lib.mask_rle([(bits, m.shape[2])], packed=True) == [r["counts"] for r in ref]


def test_one_call_mixes_sizes():
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import encode_mask_results
    masks = [_blobs(2, 800, 1333, 5), np.zeros((0, 9, 9), dtype=bool), _blobs(3, 37, 5, 6), _single(1, 1, 0),
             _blobs(1, 4097, 3, 7), np.random.default_rng(8).random((2, 100, 1030)) < 0.5]
    dev = [torch.from_numpy(m).cuda() for m in masks]
    out = encode_mask_results(dev)
    assert [len(o) for o in out] == [m.shape[0] for m in masks]
    assert out == [_ref(m) for m in masks]
    got = _lib.mask_rle([(_lib.pack_mask_bits(d), d.shape[2]) for d in dev], packed=True)
    assert got == [r["counts"] for m in masks for r in _ref(m)]


def test_empty_input_returns_empty_list():
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import encode_mask_results
    n0 = _lib.launch_count
    assert encode_mask_results(torch.zeros(0, 64, 64, dtype=torch.bool, device="cuda")) == []
    assert encode_mask_results([]) == []
    assert _lib.launch_count == n0


def test_repeatable_and_round_trips():
    from rsprompter_b200.results import coco_rle_to_mask, encode_mask_results
    m = np.concatenate([_blobs(3, 300, 257, 9), np.random.default_rng(10).random((2, 300, 257)) < 0.5])
    dev = torch.from_numpy(m).cuda()
    a, b = encode_mask_results(dev), encode_mask_results(dev)
    assert a == b
    for r, mk in zip(a, m):
        assert r["size"] == [300, 257] and isinstance(r["counts"], bytes)
        assert np.array_equal(coco_rle_to_mask(r), mk)


def test_device_record_equals_host_record():
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import ResultRecord, record_to_coco_results
    B, M, H, W = 3, 5, 96, 136
    rec = ResultRecord(B, M, (H, W), device="cuda")
    masks = np.concatenate([_blobs(B * M - 2, H, W, 11), np.random.default_rng(12).random((2, H, W)) < 0.5])
    _lib.pack_mask_bits(torch.from_numpy(masks).cuda(), bits=rec.mask_bits.view(B * M, H, W // 8))
    g = torch.Generator().manual_seed(13)
    rec.rows.copy_(torch.rand(B, M, 6, generator=g) * 50)
    rec.rows[..., 5] = torch.randint(0, 4, (B, M), generator=g).float().cuda()
    rec.counts.copy_(torch.tensor([5, 0, 3], dtype=torch.int32))
    host = rec.to_host(non_blocking=False)
    cats = {0: 1, 1: 2, 2: 3, 3: 7}
    got = record_to_coco_results(rec, image_ids=[4, 5, 6], label_to_cat=cats)
    ref = record_to_coco_results(host, image_ids=[4, 5, 6], label_to_cat=cats)
    assert len(got) == 8 and got == ref


# ---- detectors: test_cfg.rle_masks ------------------------------------------------------------------------------
def _detector(kind):
    from rsprompter_b200 import model_configs, sam_config, synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    from rsprompter_b200.registry import MODELS
    arch, nsel = sam_config.VISION_ARCHS["base"], len(SELECT_LAYERS["base"])
    if kind == "anchor":
        m = MODELS.build(model_configs.anchor_model_cfg("base", NUM_CLASSES))
        m.load_state_dict(synthetic.anchor_detector_state_dict(arch, NUM_CLASSES, nsel, seed=3), strict=True)
    elif kind == "query":
        m = MODELS.build(model_configs.query_model_cfg("base", NUM_CLASSES, prompt_shape=(20, 5)))
        m.load_state_dict(synthetic.query_detector_state_dict(arch, NUM_CLASSES, nsel, nq=20, seed=8), strict=True)
    elif kind == "maskrcnn":
        m = MODELS.build(model_configs.maskrcnn_model_cfg("base", NUM_CLASSES))
        m.load_state_dict(synthetic.maskrcnn_detector_state_dict(arch, NUM_CLASSES, nsel, seed=11), strict=True)
    elif kind == "mask2former":
        m = MODELS.build(model_configs.mask2former_model_cfg("base", NUM_CLASSES, num_queries=20))
        m.load_state_dict(synthetic.mask2former_detector_state_dict(arch, NUM_CLASSES, nsel, nq=20, seed=6), strict=True)
    else:
        m = _samdet()
    return m.cuda()


def _samdet():
    """SAMDet prompting a synthetic RSSamModel with ground-truth boxes (test_cfg.oracle_on, the reference default)."""
    from rsprompter_b200 import sam_config, synthetic
    from rsprompter_b200.registry import MODELS

    class _Boxes(torch.nn.Module):
        def predict(self, x, samples, rescale=True):
            return samples

    MODELS.register_module(name="_RleBoxesStub", module=_Boxes, force=True)
    det = MODELS.build(dict(type="SAMDet", detector=dict(type="_RleBoxesStub"),
                            segmentor=dict(type="RSSamModel", hf_pretrain_name="facebook/sam-vit-base"),
                            test_cfg=dict(oracle_on=True)))
    arch, darch = sam_config.VISION_ARCHS["base"], sam_config.SamDecoderArch()
    sd = {"shared_image_embedding.positional_embedding":
          synthetic.positional_embedding_state_dict(arch, 35)["positional_embedding"]}
    sd.update({"vision_encoder." + k: v for k, v in synthetic.vision_encoder_state_dict(arch, seed=31).items()})
    sd.update({"mask_decoder." + k: v for k, v in synthetic.mask_decoder_state_dict(darch, seed=32).items()})
    psd = synthetic.prompt_encoder_state_dict(darch, seed=34)
    g = torch.Generator().manual_seed(33)
    for i in range(4):
        psd[f"point_embed.{i}.weight"] = torch.randn(1, 256, generator=g) * 0.5
    psd["not_a_point_embed.weight"] = torch.randn(1, 256, generator=g) * 0.5
    sd.update({"prompt_encoder." + k: v for k, v in psd.items()})
    det.segmentor.sam_model.load_state_dict(sd, strict=True)
    return det


def _samples(resized):
    from rsprompter_b200.registry import InstanceData, make_data_samples
    ds = make_data_samples(2, 1024)
    if resized:      # keep-ratio resize of a 600 x 800 image, padded to the batch shape
        ds[1].set_metainfo(dict(ori_shape=(600, 800), img_shape=(768, 1024), scale_factor=(1.28, 1.28)))
    boxes = torch.tensor([[100.0, 80.0, 400.0, 300.0], [10.0, 10.0, 700.0, 500.0], [350.0, 200.0, 420.0, 260.0]])
    for d in ds:     # SAMDet's prompts; the other detectors ignore them
        d.gt_instances = InstanceData(bboxes=boxes.cuda(), labels=torch.zeros(3, dtype=torch.long).cuda())
    return ds


@pytest.fixture(scope="module", params=["anchor", "query", "maskrcnn", "mask2former", "samdet"])
def detector(request):
    return _detector(request.param)


@pytest.mark.parametrize("resized", [False, True], ids=["batch_shape", "resized_padded"])
def test_detector_rle_masks_equal_bool_masks(detector, resized):
    from rsprompter_b200.results import coco_rle_to_mask
    torch.manual_seed(4)
    x = torch.randn(2, 3, 1024, 1024).cuda()
    detector.test_cfg["rle_masks"] = False
    ref = detector.predict(x, _samples(resized))
    detector.test_cfg["rle_masks"] = True
    try:
        out = detector.predict(x, _samples(resized))
    finally:
        detector.test_cfg["rle_masks"] = False
    total = 0
    for r, o in zip(ref, out):
        rp, op = r.pred_instances, o.pred_instances
        for k in ("bboxes", "scores", "labels"):
            assert torch.equal(getattr(rp, k), getattr(op, k)), k
        ori = [int(v) for v in r.metainfo["ori_shape"][:2]]
        assert isinstance(op.masks, list) and len(op.masks) == rp.masks.shape[0]
        for rle, mk in zip(op.masks, rp.masks.cpu().numpy()):
            assert rle["size"] == ori and isinstance(rle["counts"], bytes)
            assert np.array_equal(coco_rle_to_mask(rle), mk)
        total += len(op.masks)
    assert total > 0
