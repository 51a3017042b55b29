"""Mask polygons on the GPU (csrc/contours.cu through _lib.mask_contours) against cv2.findContours(RETR_CCOMP) point for
point, in list order and hierarchy, in both approximation modes: on every 4 x 4 mask, odd widths, single rows and
columns, structured 1024^2 masks, placed and union canvases, with repeat calls and split calls; then the public
entry points that use it: bitmap_to_polygon, record_polygons, the large-scene and segment-everything polygons and the
CLIs' GeoJSON output."""
import json

import numpy as np
import pytest
import torch

from rsprompter_b200 import _lib, results

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

MODES = (_lib.CHAIN_APPROX_NONE, _lib.CHAIN_APPROX_SIMPLE)


def _cv2(mask, approx):
    c, h = cv2.findContours(np.ascontiguousarray(mask).astype(np.uint8), cv2.RETR_CCOMP, approx)
    return [x.reshape(-1, 2) for x in c], h


def _same(got, want, what=""):
    (gc, gh), (wc, wh) = got, want
    assert len(gc) == len(wc), f"{what}: {len(gc)} contours, cv2 {len(wc)}"
    for k, (a, b) in enumerate(zip(gc, wc)):
        assert a.dtype == np.int32 and np.array_equal(a, b), f"{what}: contour {k}\n{a}\n{b}"
    if wh is None:
        assert gh is None, what
    else:
        assert gh is not None and np.array_equal(gh, wh), f"{what}: hierarchy\n{gh}\n{wh}"


def _bits(masks):
    """bool [n, H, W] -> bit rows uint8 [n, H, ceil(W/8)] on the GPU."""
    return torch.from_numpy(np.packbits(masks, axis=-1, bitorder="little")).cuda()


def _plain(masks, approx, **kw):
    n, H, W = masks.shape
    bits = _bits(masks)
    ld = bits.shape[-1]
    return _lib.mask_contours([bits], [(H, W, [(0, j * H * ld, ld, H, H, W, 0, 0)]) for j in range(n)], approx, **kw)


@pytest.mark.parametrize("approx", MODES)
def test_every_4x4_mask_in_one_call(approx):
    codes = np.arange(1 << 16)
    masks = ((codes[:, None] >> np.arange(16)) & 1).astype(bool).reshape(-1, 4, 4)
    got = _plain(masks, approx)
    for m, g in zip(masks, got):
        _same(g, _cv2(m, approx), str(m.astype(int)))


@pytest.mark.parametrize("approx", MODES)
@pytest.mark.parametrize("hw", [(1, 1), (1, 37), (53, 1), (7, 13), (29, 31), (33, 65), (64, 100), (17, 250)])
def test_odd_shapes(approx, hw):
    rng = np.random.default_rng(hw[0] * 1000 + hw[1])
    masks = np.stack([rng.random(hw) < d for d in (0.0, 0.2, 0.5, 0.7, 0.9, 1.0)])
    for m, g in zip(masks, _plain(masks, approx)):
        _same(g, _cv2(m, approx), f"{hw}")


@pytest.mark.parametrize("approx", MODES)
def test_structured_1024(approx):
    from test_small_regions_gpu import _contents
    masks = _contents(1024, 1024, 3)
    got = _plain(masks, approx)
    for k, (m, g) in enumerate(zip(masks, got)):
        _same(g, _cv2(m, approx), f"content {k}")


def _placed_cases(seed):
    """Sources of random masks and union canvases over them: x0 % 8 != 0, overlapping parts, parts at the canvas edges;
    -> (sources, canvases, host canvases)."""
    rng = np.random.default_rng(seed)
    srcs = [rng.random((6, 40, 56)) < 0.55, rng.random((3, 70, 33)) < 0.4]
    bits = [_bits(s) for s in srcs]
    H, W = 120, 150
    canvases, host = [], []
    for c in range(24):
        k = 1 + c % 4
        parts, canvas = [], np.zeros((H, W), bool)
        for _ in range(k):
            si = int(rng.integers(2))
            j = int(rng.integers(srcs[si].shape[0]))
            sh, sw = srcs[si].shape[1:]
            h, w = int(rng.integers(1, sh + 1)), int(rng.integers(1, sw + 1))
            y0 = int(rng.integers(0, H - h + 1)) if c % 3 else H - h      # some flush with the bottom / right edges
            x0 = int(rng.integers(0, W - w + 1)) if c % 5 else W - w
            ld = bits[si].shape[-1]
            parts.append((si, j * sh * ld, ld, sh, h, w, y0, x0))
            canvas[y0:y0 + h, x0:x0 + w] |= srcs[si][j, :h, :w]
        canvases.append((H, W, parts))
        host.append(canvas)
    return bits, canvases, host


@pytest.mark.parametrize("approx", MODES)
def test_placed_and_union_canvases(approx):
    bits, canvases, host = _placed_cases(7)
    assert any(p[7] % 8 for _, _, pl in canvases for p in pl)
    got = _lib.mask_contours(bits, canvases, approx)
    for k, (canvas, g) in enumerate(zip(host, got)):
        _same(g, _cv2(canvas, approx), f"canvas {k}")


def test_two_calls_and_split_calls_agree():
    from test_small_regions_gpu import _contents
    masks = _contents(256, 200, 5)
    bits, canvases, _ = _placed_cases(11)
    for approx in MODES:
        a = _plain(masks, approx)
        b = _plain(masks, approx)
        c = _plain(masks, approx, ws_bound=1)                      # one canvas per call
        for x, y, z in zip(a, b, c):
            _same(x, y)
            _same(x, z)
        u = _lib.mask_contours(bits, canvases, approx)
        v = _lib.mask_contours(bits, canvases, approx, ws_bound=300_000)
        for x, y in zip(u, v):
            _same(x, y)


def test_bitmap_to_polygon_equals_mmdet():
    """mmdet's bitmap_to_polygon (mmdet/structures/mask/structures.py:1166-1194), restated with cv2, per mask."""
    def mmdet_bitmap_to_polygon(bitmap):
        outs = cv2.findContours(np.ascontiguousarray(bitmap).astype(np.uint8), cv2.RETR_CCOMP, cv2.CHAIN_APPROX_NONE)
        contours, hierarchy = outs[-2], outs[-1]
        if hierarchy is None:
            return [], False
        with_hole = (hierarchy.reshape(-1, 4)[:, 3] >= 0).any()
        return [c.reshape(-1, 2) for c in contours], with_hole

    from test_small_regions_gpu import _contents
    masks = _contents(96, 77, 2)
    for dtype in (torch.bool, torch.uint8):
        got = results.bitmap_to_polygon(torch.from_numpy(masks).to(dtype).cuda())
        assert len(got) == len(masks)
        for m, (c, hole) in zip(masks, got):
            wc, wh = mmdet_bitmap_to_polygon(m)
            assert hole == wh and len(c) == len(wc)
            for a, b in zip(c, wc):
                assert np.array_equal(a, b)


# ---- the pipelines ------------------------------------------------------------------------------------------------
from test_scene_mask_generation_gpu import _run, blobs, sam  # noqa: E402,F401  (module fixtures)


def _same_as_rle(polygons, rles, approx=_lib.CHAIN_APPROX_SIMPLE):
    """Each mask's polygons equal cv2 on the mask decoded from its RLE."""
    assert len(polygons) == len(rles) > 0
    for k, (poly, rle) in enumerate(zip(polygons, rles)):
        _same(poly, _cv2(results.coco_rle_to_mask(rle), approx), f"mask {k}")


def test_record_polygons_of_a_detector_record():
    from test_large_image_gpu import _model, _scene

    from rsprompter_b200.large_image import run_tiles
    records, _ = run_tiles(_model("query"), _scene(1024, 1024, seed=3), batch_size=2)
    rec = records[0]
    got = results.record_polygons(rec)
    insts = rec.instances()
    assert len(got) == len(insts) and sum(len(g) for g in got) > 0
    for polys, inst in zip(got, insts):
        masks = inst["masks"].cpu().numpy()
        assert len(polys) == len(masks)
        for (c, hole), m in zip(polys, masks):
            wc, wh = _cv2(m, cv2.CHAIN_APPROX_NONE)
            assert hole == (wh is not None and bool((wh.reshape(-1, 4)[:, 3] >= 0).any()))
            assert len(c) == len(wc) and all(np.array_equal(a, b) for a, b in zip(c, wc))


def test_predict_large_image_greedy_nmm_polygons():
    from test_large_image_gpu import _model, _scene

    from rsprompter_b200.large_image import predict_large_image
    model = _model("query")
    scene = _scene(1100, 1500, seed=1)
    ds = predict_large_image(model, scene, merge_iou_thr=0.3, merge_nms_type="greedy_nmm", output_polygons=True)
    _same_as_rle(ds.pred_instances.polygons, ds.pred_instances.masks)
    plain = predict_large_image(model, scene, merge_iou_thr=0.3, merge_nms_type="greedy_nmm")
    assert "polygons" not in plain.pred_instances
    assert [m["counts"] for m in plain.pred_instances.masks] == [m["counts"] for m in ds.pred_instances.masks]


def test_generate_scene_masks_polygons(sam, monkeypatch, blobs):
    res = _run(sam, monkeypatch, blobs, batch_size=4, output_polygons=True)
    _same_as_rle(res["polygons"], res["rle"])
    plain = _run(sam, monkeypatch, blobs, batch_size=4)
    assert "polygons" not in plain and [r["counts"] for r in plain["rle"]] == [r["counts"] for r in res["rle"]]


def _check_geojson(fc, rows):
    """A FeatureCollection against the COCO-format rows of the same run: properties and geometry per row."""
    from rsprompter_b200.geojson import multipolygon
    assert fc["type"] == "FeatureCollection" and len(fc["features"]) == len(rows) > 0
    for f, row in zip(fc["features"], rows):
        assert f["properties"] == {k: v for k, v in row.items() if k != "segmentation"}
        mask = results.coco_rle_to_mask(row["segmentation"])
        want = multipolygon(*_cv2(mask, cv2.CHAIN_APPROX_SIMPLE))
        assert f["geometry"] == json.loads(json.dumps(want))


def test_large_image_cli_geojson(tmp_path):
    from test_large_image_gpu import _model, _model_cfg, _scene

    from rsprompter_b200.large_image import main
    model = _model("query")
    cfg = tmp_path / "cfg.py"
    cfg.write_text("model = " + repr(_model_cfg("query")) + "\n")
    ckpt = tmp_path / "model.pth"
    torch.save(dict(state_dict=model.state_dict()), ckpt)
    img = tmp_path / "scene.png"
    cv2.imwrite(str(img), _scene(700, 900, seed=7))
    coco, geo = tmp_path / "results.json", tmp_path / "results.geojson"
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(coco)])
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(geo), "--out-format", "geojson"])
    _check_geojson(json.loads(geo.read_text()), json.loads(coco.read_text()))


def test_mask_generation_cli_geojson(sam, tmp_path):
    from rsprompter_b200 import mask_generation as mg
    rgb = torch.from_numpy(np.random.default_rng(9).integers(0, 255, (3, 240, 320), dtype=np.uint8))
    path = tmp_path / "img.png"
    cv2.imwrite(str(path), rgb.permute(1, 2, 0).flip(-1).numpy())
    ckpt = tmp_path / "sam.pth"
    torch.save(sam["sd"], ckpt)
    args = [str(path), "--arch", "base", "--checkpoint", str(ckpt), "--points-per-side", "4", "--pred-iou-thresh", "0",
            "--stability-score-thresh", "0"]
    coco, geo = tmp_path / "masks.json", tmp_path / "masks.geojson"
    mg.main(args + ["--out", str(coco)])
    mg.main(args + ["--out", str(geo), "--out-format", "geojson"])
    _check_geojson(json.loads(geo.read_text()), json.loads(coco.read_text()))
