"""Coarse layers of segment-everything over a whole scene on the GPU: rsp_resize_aa_pad_u8 against torchvision's
antialiased uint8 resize and against SamImageProcessor; generate_scene_masks(coarse_patch_sizes=...) against the
base-only call, against oracle.restate_scene_layers on structured decoder outputs (helpers copied from
test_scene_mask_generation_gpu.py), on an object larger than the overlap, with small mask groups, its host
synchronisations and the CLI."""
import json
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SCENE = (1536, 2048)         # six 1024 x 1024 windows at the default overlap
COARSE = (1600, 4096)        # two 1600-px windows, then the whole scene
MEAN = tuple(255.0 * m for m in (0.485, 0.456, 0.406))
STD = tuple(255.0 * s for s in (0.229, 0.224, 0.225))


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


def _tv(img, size):
    from torchvision.transforms.v2 import functional as tvF
    return tvF.resize(img.cpu(), list(size), interpolation=tvF.InterpolationMode.BILINEAR, antialias=True)


def _normalised(u8, hp, wp, pad=MEAN):
    """fp32 (u - mean) / std of uint8 [3, h, w] padded to [3, hp, wp] with the normalised pad, as the kernel forms it."""
    m = torch.tensor(MEAN, dtype=torch.float32)[:, None, None]
    s = torch.tensor(STD, dtype=torch.float32)[:, None, None]
    out = ((torch.tensor(pad, dtype=torch.float32)[:, None, None] - m) / s).expand(3, hp, wp).clone()
    out[:, :u8.shape[1], :u8.shape[2]] = (u8.float() - m) / s
    return out


# ------------------------------------------------------------------------------------------------ the kernel
SIZE_PAIRS = [((2048, 1500), (1024, 750)), ((1500, 900), (1024, 614)), ((600, 800), (768, 1024)),
              ((1037, 2311), (460, 1024)), ((333, 517), (1024, 1024)), ((500, 700), (500, 350)),
              ((97, 131), (97, 131))]


@pytest.mark.parametrize("src, dst", SIZE_PAIRS)
def test_kernel_is_torchvision_byte_for_byte(src, dst):
    from rsprompter_b200 import _lib
    img = torch.from_numpy(np.random.default_rng(sum(src)).integers(0, 256, (3, *src), dtype=np.uint8))
    out = torch.full((1, 3, 1024, 1024), float("nan"), device="cuda")
    _lib.resize_aa_pad_u8([img.cuda()], [dst], out, MEAN, STD, False, MEAN)
    assert _same(out[0].cpu(), _normalised(_tv(img, dst), 1024, 1024))


def test_strided_views_of_a_device_scene_in_a_mixed_batch_with_pad():
    """Windows of a permuted HWC scene read in place, of four sizes in one launch, channels swapped, and pixels
    outside each resized image equal to the normalised pad value."""
    from rsprompter_b200 import _lib
    scene = _image((3000, 4100), 7)
    dev = scene.permute(1, 2, 0).contiguous().cuda().permute(2, 0, 1)          # [3, H, W] view of HWC memory
    boxes = [(0, 0, 4100, 3000), (100, 50, 2148, 1586), (3000, 2000, 4100, 3000), (10, 20, 900, 2900)]
    sizes = [(749, 1024), (768, 1024), (931, 1024), (1024, 313)]
    pad = (12.5, 200.0, 3.0)
    out = torch.empty(len(boxes), 3, 1024, 1024, device="cuda")
    views = [dev[:, y0:y1, x0:x1] for x0, y0, x1, y1 in boxes]
    _lib.resize_aa_pad_u8(views, sizes, out, MEAN, STD, True, pad)
    for b, ((x0, y0, x1, y1), hw) in enumerate(zip(boxes, sizes)):
        ref = _tv(scene[:, y0:y1, x0:x1], hw).flip(0)
        assert _same(out[b].cpu(), _normalised(ref, 1024, 1024, pad[::-1])), b


def test_a_size_beyond_the_pad_is_refused():
    from rsprompter_b200 import _lib
    img = torch.zeros(3, 64, 64, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.RspError, match="inside the pad size"):
        _lib.resize_aa_pad_u8([img], [(40, 2000)], torch.empty(1, 3, 1024, 1024, device="cuda"), MEAN, STD, False, MEAN)


@pytest.mark.parametrize("hw", [(1500, 900), (4096, 4096)])
def test_kernel_batch_is_sam_image_processor(hw):
    from transformers import SamImageProcessor

    from rsprompter_b200 import _lib
    from rsprompter_b200.mask_generation import preprocess_shape
    img = _image(hw, 11)
    ref = SamImageProcessor()(images=img, return_tensors="pt")["pixel_values"][0]
    out = torch.empty(1, 3, 1024, 1024, device="cuda")
    _lib.resize_aa_pad_u8([img.cuda()], [preprocess_shape(hw, 1024)], out, MEAN, STD, False, MEAN)
    diff = (out[0].cpu() - ref).abs().max().item()
    hf_mean = torch.tensor((0.485, 0.456, 0.406), dtype=torch.float32) * 255
    hf_std = torch.tensor((0.229, 0.224, 0.225), dtype=torch.float32) * 255
    if torch.equal(hf_mean, torch.tensor(MEAN, dtype=torch.float32)) and \
            torch.equal(hf_std, torch.tensor(STD, dtype=torch.float32)):
        assert diff == 0.0
    else:                       # the constants round differently: the grey levels are still the same bytes
        print(f"SamImageProcessor vs kernel at {hw}: max |diff| = {diff:.3e}")
        assert diff < 1e-5


# ------------------------------------------------------------------------------------------------ layers
N_SIDE = 6
N_PTS = N_SIDE * N_SIDE


def _blobs(n_tiles, seed):
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
    """Serves seeded outputs in place of the mask decoder, prompt by prompt across windows in run order."""

    def __init__(self, low, iou):
        self.low, self.iou, self.served = low.cuda(), iou.cuda(), 0

    def __call__(self, emb_rows, pos_rows, sparse, hw, **kw):
        q0 = self.served
        self.served += sparse.shape[0]
        return self.low[q0:self.served], self.iou[q0:self.served]


def _kw(low, iou, crops, hw):
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
    from rsprompter_b200.mask_generation import scene_layer_windows
    layers = scene_layer_windows(SCENE, 1024, 0.25, COARSE)
    assert [len(c) for _, c in layers] == [6, 2, 1]
    n = sum(len(c) for _, c in layers)
    low, iou = _blobs(n, seed=5)
    return dict(low=low, iou=iou, layers=layers, kw=_kw(low, iou, layers[0][1], SCENE), scene=_image(SCENE, 3))


def _run(sam, monkeypatch, blobs, n_windows, **kw):
    from rsprompter_b200 import mask_generation as mg
    dec = _Decoder(blobs["low"], blobs["iou"])
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    res = mg.generate_scene_masks(sam["model"], blobs["scene"], points_per_side=N_SIDE, points_per_batch=64,
                                  **dict(blobs["kw"], **kw))
    assert dec.served == n_windows * N_PTS
    return res


def _rows_equal(a, b, n=None):
    sl = slice(0, n)
    assert [x["counts"] for x in a["rle"][sl]] == [x["counts"] for x in b["rle"]]
    for k in ("scores", "stability_scores", "boxes", "points", "tiles", "crop_boxes"):
        assert _same(a[k][sl], b[k]), k
    assert torch.equal(a["candidates"][sl], b["candidates"])


def test_no_coarse_layer_is_the_call_without_the_keyword(sam, monkeypatch, blobs):
    a = _run(sam, monkeypatch, blobs, 6, batch_size=4)
    b = _run(sam, monkeypatch, blobs, 6, batch_size=4, coarse_patch_sizes=())
    assert len(a["rle"]) > 0
    _rows_equal(a, b)
    assert a["layers"].eq(0).all() and a["layers"].device.type == "cuda" and len(a["layers"]) == len(a["rle"])


@pytest.mark.parametrize("area", [0.0, 150.5])
def test_layers_match_the_oracle_and_the_base_rows_are_a_prefix(sam, monkeypatch, blobs, area):
    from oracle import restate_mask_generation as R
    from oracle import restate_scene_layers as L
    from oracle import restate_scene_mask_generation as O
    from rsprompter_b200.mask_generation import preprocess_shape
    from rsprompter_b200.results import coco_rle_to_mask
    low, iou, kw = blobs["low"], blobs["iou"], blobs["kw"]
    wins, per_layer, g = [], [], 0
    for l, crops in blobs["layers"]:
        lw, pts = [], []
        for t, cb in enumerate(crops):
            whw = (cb[3] - cb[1], cb[2] - cb[0])
            sl = slice((g + t) * N_PTS, (g + t + 1) * N_PTS)
            lw.append(O.generate_window(low[sl], iou[sl], cb, SCENE, preprocess_shape(whw, 1024),
                                        min_mask_region_area=area, **kw))
            pts.append(R.grid_prompts(N_SIDE, whw)[0])
        m = O.merge(lw, crops, pts, kw["crops_nms_thresh"])
        m["window"] = m["tiles"] + g
        per_layer.append((l, m))
        wins += lw
        g += len(crops)
    merged = L.merge_layers(per_layer, kw["crops_nms_thresh"])
    assert set(merged["layers"].tolist()) == {0, 1, 2}            # every layer contributes a row
    assert len(merged["layers"]) < sum(len(m["tiles"]) for _, m in per_layer)   # and the cross-layer NMS drops some
    base = _run(sam, monkeypatch, blobs, 6, batch_size=4, min_mask_region_area=area)
    got = _run(sam, monkeypatch, blobs, 9, batch_size=4, min_mask_region_area=area, coarse_patch_sizes=COARSE)
    _rows_equal(got, base, len(base["rle"]))
    assert got["layers"][:len(base["rle"])].eq(0).all()
    assert torch.equal(got["layers"].cpu(), merged["layers"])
    assert torch.equal(got["tiles"].cpu(), merged["tiles"])
    assert torch.equal(got["candidates"], merged["candidates"])
    assert torch.equal(got["scores"].cpu(), merged["scores"])
    assert torch.equal(got["boxes"].cpu(), merged["boxes"])
    assert torch.equal(got["points"].cpu(), merged["points"])
    crops_all = [cb for _, c in blobs["layers"] for cb in c]
    assert torch.equal(got["crop_boxes"].cpu(), torch.tensor(crops_all)[merged["window"]])
    eps = 1e-4 * max(1.0, low.abs().max().item())
    for i, (w, rank, c) in enumerate(zip(merged["window"].tolist(), merged["rank"].tolist(),
                                         merged["candidates"].tolist())):
        cb = crops_all[w]
        whw = (cb[3] - cb[1], cb[2] - cb[0])
        v = R.upscale(low[w * N_PTS + c // 3, c % 3], whw, preprocess_shape(whw, 1024))
        tie = O.uncrop(((v - 0.0).abs() <= eps)[None], cb, SCENE)[0]
        ref = O.uncrop(wins[w]["masks"][rank][None], cb, SCENE)[0]
        m = torch.from_numpy(coco_rle_to_mask(got["rle"][i])).bool()
        assert got["rle"][i]["size"] == list(SCENE)
        assert torch.equal(m & ~tie, ref & ~tie), i


@pytest.mark.parametrize("area", [0.0, 150.5])
def test_small_mask_groups_give_the_same_result(sam, monkeypatch, blobs, area):
    """A scene whose coarse masks do not fit one group: groups of three whole-scene masks at most."""
    from rsprompter_b200 import mask_generation as mg
    ref = _run(sam, monkeypatch, blobs, 9, batch_size=2, min_mask_region_area=area, coarse_patch_sizes=COARSE)
    per = SCENE[0] * ((SCENE[1] + 15) // 16 * 2)
    monkeypatch.setattr(mg, "COARSE_MASK_BYTES", 3 * per)
    held = []
    paste = mg._paste

    def spy(cand, b, ci, *a):
        bits = paste(cand, b, ci, *a)
        if bits.shape[1] == SCENE[0]:                           # a coarse window's masks
            held.append(bits.numel())
        return bits
    monkeypatch.setattr(mg, "_paste", spy)
    got = _run(sam, monkeypatch, blobs, 9, batch_size=2, min_mask_region_area=area, coarse_patch_sizes=COARSE)
    assert len(held) > 3 and max(held) <= 3 * per
    _rows_equal(got, ref)
    assert torch.equal(got["layers"], ref["layers"])


def test_an_object_larger_than_the_overlap_is_found_by_a_coarse_layer(sam, monkeypatch):
    """One disc of radius 400 px across the seams of every base window: the edge rule drops it in each, and the
    whole-scene layer returns it."""
    from rsprompter_b200 import mask_generation as mg
    cx, cy, rad = 1000.0, 768.0, 400.0
    layers = mg.scene_layer_windows(SCENE, 1024, 0.25, (4096,))
    lows = []
    for _, crops in layers:
        for x0, y0, x1, y1 in crops:
            h, w = y1 - y0, x1 - x0
            nh, nw = mg.preprocess_shape((h, w), 1024)
            u = (torch.arange(256.0) * 4 + 1.5)
            ys, xs = u[:, None] * h / nh + y0, u[None, :] * w / nw + x0
            disc = (rad - ((ys - cy) ** 2 + (xs - cx) ** 2).sqrt()).clamp(-8, 8)
            low = torch.full((N_PTS, 3, 256, 256), -8.0)
            low[0, 0] = disc
            lows.append(low)
    low = torch.cat(lows)
    iou = torch.zeros(low.shape[0], 3)
    iou[0::N_PTS, 0] = 0.99
    kw = dict(points_per_side=N_SIDE, pred_iou_thresh=0.5, stability_score_thresh=0.0)
    scene = _image(SCENE, 9)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", _Decoder(low, iou))
    base = mg.generate_scene_masks(sam["model"], scene, **kw)
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", _Decoder(low, iou))
    got = mg.generate_scene_masks(sam["model"], scene, coarse_patch_sizes=(4096,), **kw)
    assert len(base["rle"]) == 0
    assert len(got["rle"]) == 1 and got["layers"].tolist() == [1] and got["tiles"].tolist() == [0]
    x0, y0, x1, y1 = got["boxes"][0].tolist()
    assert abs(x0 - (cx - rad)) < 8 and abs(x1 - (cx + rad)) < 8 and abs(y0 - (cy - rad)) < 8 and abs(y1 - (cy + rad)) < 8


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
def test_host_synchronisations_per_batch_per_layer_and_one_across_layers(sam, monkeypatch, blobs, area):
    """Each batch of windows, base or coarse, costs what it costs without layers; then one merge per layer and one
    cross-layer NMS."""
    from rsprompter_b200 import mask_generation as mg
    scene = blobs["scene"].cuda()
    kw = dict(blobs["kw"], points_per_side=N_SIDE, points_per_batch=64, min_mask_region_area=area)

    decoders = iter([_Decoder(blobs["low"], blobs["iou"]) for _ in range(6)])        # built outside the count

    def call(b, coarse):
        monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", next(decoders))
        return mg.generate_scene_masks(sam["model"], scene, batch_size=b, coarse_patch_sizes=coarse, **kw)
    per_batch = 3 + (area > 0)
    for b in (2, 3):
        res = call(b, COARSE)
        assert set(res["layers"].tolist()) == {0, 1, 2}
        n_base = _host_syncs(lambda: call(b, ()))
        assert n_base == per_batch * (6 // b) + 1
        n = _host_syncs(lambda: call(b, COARSE))
        assert n == per_batch * (6 // b + 1 + 1) + 3 + 1, (n, b)


def test_cli_writes_the_layer_with_the_flag(sam, monkeypatch, blobs, tmp_path):
    import cv2

    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.sam_decoder import SamMaskDecoderB200
    path = tmp_path / "scene.png"
    cv2.imwrite(str(path), blobs["scene"].permute(1, 2, 0).flip(-1).numpy())
    ckpt = tmp_path / "sam.pth"
    torch.save(sam["sd"], ckpt)
    dec = _Decoder(blobs["low"], blobs["iou"])
    monkeypatch.setattr(SamMaskDecoderB200, "decode", lambda self, *a, **kw: dec(*a, **kw))
    monkeypatch.setattr(sam["model"].sam_model.mask_decoder, "decode", dec)
    out = tmp_path / "masks.json"
    kw = blobs["kw"]
    mg.main([str(path), "--arch", "base", "--checkpoint", str(ckpt), "--points-per-side", str(N_SIDE),
             "--pred-iou-thresh", str(kw["pred_iou_thresh"]), "--stability-score-thresh",
             str(kw["stability_score_thresh"]), "--crops-nms-thresh", str(kw["crops_nms_thresh"]),
             "--patch-size", "1024", "--coarse-patch-sizes", *map(str, COARSE), "--out", str(out)])
    rows = json.loads(out.read_text())
    dec.served = 0
    ref = mg.generate_scene_masks(sam["model"], blobs["scene"], points_per_side=N_SIDE, coarse_patch_sizes=COARSE, **kw)
    assert len(rows) == len(ref["rle"]) > 0
    assert [r["layer"] for r in rows] == ref["layers"].tolist()
    for row, r in zip(rows, ref["rle"]):
        assert set(row) == {"segmentation", "bbox", "predicted_iou", "stability_score", "point_coords", "crop_box",
                            "layer"}
        assert row["segmentation"]["counts"] == r["counts"].decode()
