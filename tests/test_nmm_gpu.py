"""Greedy non-maximum merging of large scenes on the device: the union RLE encoder against results.mask_to_coco_rle
of the OR'd canvas, merge_tile_records(nms_type='greedy_nmm') against oracle.restate_nmm, the seam case, and
predict_large_image(merge_nms_type='greedy_nmm') end to end against a composition of host records, the oracle merge,
the OR of sahi's shift_masks and the host RLE."""
import json
import warnings

import numpy as np
import pytest
import torch

from oracle import restate_large_image as oracle_li
from oracle import restate_nmm as oracle
from test_large_image_gpu import _blobs, _model, _model_cfg, _scene

pytestmark = pytest.mark.gpu

NUM_CLASSES = 10


# ---- union RLE ----------------------------------------------------------------------------------------------------
_P = 64
_T = _blobs(6, _P, _P, 20)
_NOISE = np.random.default_rng(21).random((2, _P, _P)) < 0.5
_ONES = np.ones((_P, _P), bool)
_ZEROS = np.zeros((_P, _P), bool)
UNION = {   # canvas (H, W), parts [(tile, (y0, x0))]
    "one": ((200, 300), [(_T[0], (70, 90))]),
    "horizontal_overlap": ((200, 300), [(_T[0], (50, 100)), (_NOISE[0], (50, 140))]),
    "vertical_overlap": ((200, 300), [(_T[1], (50, 100)), (_T[2], (90, 100))]),
    "corner_2x2": ((200, 300), [(_T[0], (10, 10)), (_T[1], (10, 50)), (_NOISE[1], (50, 10)), (_ONES, (50, 50))]),
    "full_height": ((64, 300), [(_NOISE[0], (0, 20)), (_T[3], (0, 60)), (_ONES, (0, 236))]),
    "full_height_stacked": ((100, 300), [(_T[4], (0, 30)), (_ONES, (36, 50))]),     # the rectangle spans H
    "full_height_gap": ((64, 300), [(_ONES, (0, 0)), (_ONES, (0, 100))]),           # an all-zero run of columns
    "bottom_right_edges": ((200, 300), [(_T[5], (136, 236)), (_ONES, (120, 200)), (_NOISE[1], (136, 0))]),
    "w_not_multiple_of_8": ((203, 301), [(_T[0], (139, 237)), (_NOISE[0], (100, 230))]),
    "disjoint": ((200, 300), [(_T[1], (10, 10)), (_T[2], (120, 200))]),
    "all_zero": ((200, 300), [(_ZEROS, (10, 10)), (_ZEROS, (40, 30))]),
    "zero_and_ones_at_bottom": ((200, 300), [(_ZEROS, (10, 10)), (_ONES, (136, 30))]),
    "overhang": ((40, 90), [(_T[2], (0, 0)), (_NOISE[1], (0, 40))]),               # visible parts clipped
    "same_place_twice": ((200, 300), [(_T[3], (70, 90)), (_T[3], (70, 90))]),
}


def _canvas(parts, hw):
    H, W = hw
    c = np.zeros((H, W), dtype=bool)
    for t, (y0, x0) in parts:
        h, w = min(t.shape[0], H - y0), min(t.shape[1], W - x0)
        c[y0:y0 + h, x0:x0 + w] |= t[:h, :w]
    return c


def _encode_union(cases, packed, src_index=0, sources=None):
    """One union call over every (canvas, parts) in ``cases``; each part's tile is a mask of one source tensor."""
    from rsprompter_b200 import _lib
    tiles = [t for _, parts in cases for t, _ in parts]
    P = tiles[0].shape[0]
    src = torch.from_numpy(np.stack(tiles)).cuda()
    src = _lib.pack_mask_bits(src) if packed else src
    ld = src.shape[2]
    canvases, j = [], 0
    for (H, W), parts in cases:
        pl = []
        for t, (y0, x0) in parts:
            pl.append((src_index, j * P * ld, ld, P, min(P, H - y0), min(P, W - x0), y0, x0))
            j += 1
        canvases.append((H, W, pl))
    if sources is None:
        return _lib.mask_rle_union([src], canvases, packed=packed)
    sources.append(src)
    return canvases


@pytest.mark.parametrize("packed", [False, True], ids=["bool", "bits"])
@pytest.mark.parametrize("name", list(UNION))
def test_union_rle_equals_canvas_rle(name, packed):
    from rsprompter_b200.results import mask_to_coco_rle
    hw, parts = UNION[name]
    ref = mask_to_coco_rle(_canvas(parts, hw))["counts"]
    assert _encode_union([UNION[name]], packed) == [ref]


@pytest.mark.parametrize("packed", [False, True], ids=["bool", "bits"])
def test_union_of_one_part_is_the_placed_string(packed):
    from rsprompter_b200 import _lib
    cases = [((200, 300), [(t, yx)]) for t, yx in [(_T[0], (0, 0)), (_NOISE[0], (136, 236)), (_ONES, (70, 90))]]
    cases += [((64, 300), [(_NOISE[1], (0, 100))]), ((203, 301), [(_T[1], (139, 237))]), ((33, 45), [(_ONES, (0, 0))])]
    tiles = torch.from_numpy(np.stack([p[0][0] for _, p in cases])).cuda()
    src = _lib.pack_mask_bits(tiles) if packed else tiles
    ld = src.shape[2]
    pl = [(j * _P * ld, ld, _P, min(_P, H - y0), min(_P, W - x0), H, W, y0, x0)
          for j, ((H, W), [(_, (y0, x0))]) in enumerate(cases)]
    assert _encode_union(cases, packed) == _lib.mask_rle_placed([(src, pl)], packed=packed)


@pytest.mark.parametrize("packed", [False, True], ids=["bool", "bits"])
def test_union_rle_two_sources_of_different_tile_sizes(packed):
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import mask_to_coco_rle
    t61 = _blobs(3, 61, 61, 22)
    cases64 = list(UNION.values())
    cases61 = [((100, 170), [(t61[0], (39, 109)), (t61[1], (20, 80))]), ((61, 500), [(t61[2], (0, 3))])]
    sources = []
    c61 = _encode_union(cases61, packed, src_index=0, sources=sources)
    c64 = _encode_union(cases64, packed, src_index=1, sources=sources)
    # one canvas mixing both sources
    mixed = (150, 210, [c61[0][2][0], c64[1][2][1]])
    got = _lib.mask_rle_union(sources, c61 + c64 + [mixed], packed=packed)
    ref = [mask_to_coco_rle(_canvas(parts, hw))["counts"] for hw, parts in cases61 + cases64]
    ref.append(mask_to_coco_rle(_canvas([(t61[0], (39, 109)), (_NOISE[0], (50, 140))], (150, 210)))["counts"])
    assert got == ref
    assert _lib.mask_rle_union(sources, c61 + c64 + [mixed], packed=packed) == got      # deterministic


def test_union_rle_large_canvas():
    """Two overlapping 1024^2 blob parts in a 20 000 x 20 000 scene (the canvas never exists on the device)."""
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import mask_to_coco_rle
    tiles = _blobs(2, 1024, 1024, 23)
    H = W = 20000
    org = [(12000, 18200), (12500, 18976)]
    src = _lib.pack_mask_bits(torch.from_numpy(tiles).cuda())
    parts = [(0, j * 1024 * 128, 128, 1024, 1024, 1024, y0, x0) for j, (y0, x0) in enumerate(org)]
    got = _lib.mask_rle_union([src], [(H, W, parts)], packed=True)[0]
    assert got == mask_to_coco_rle(_canvas(list(zip(tiles, org)), (H, W)))["counts"]


# ---- the merge against the oracle ---------------------------------------------------------------------------------
def _records(n_tiles, P, M, seed, batch=4, full=False, bits=False):
    """Seeded ResultRecords of n_tiles tiles (batch images each, the last one partly used) with distinct scores;
    ``bits``: random mask bits in every slot."""
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
        if bits:
            rec.mask_bits.copy_(torch.randint(0, 256, rec.mask_bits.shape, generator=g, dtype=torch.uint8))
        recs.append(rec)
    return recs


def _host_tiles(recs, origins):
    tiles, offs, src = [], [], []
    for r, (rec, org) in enumerate(zip(recs, origins)):
        host = rec.to_host(non_blocking=False)
        inst = host.instances()
        for b, o in enumerate(org):
            tiles.append(inst[b])
            offs.append(o)
            src += [(r, b, s) for s in range(int(host.counts[b]))]
    return tiles, offs, torch.tensor(src, dtype=torch.int64).view(-1, 3)


def _oracle_nmm(recs, origins, hw, thr, metric, P, score_thr=0.0):
    tiles, offs, src = _host_tiles(recs, origins)
    boxes_only = [{k: t[k] for k in ("bboxes", "scores", "labels")} for t in tiles]
    merged, groups = oracle.merge_results_by_nmm(boxes_only, offs, hw, thr, metric, patch=P, score_thr=score_thr)
    members = src[torch.tensor([i for g in groups for i in g], dtype=torch.int64)]
    offsets = torch.tensor([0] + np.cumsum([len(g) for g in groups]).tolist(), dtype=torch.int64)
    return merged, groups, members, offsets, tiles, offs


def _assert_merge_equal(got, merged, groups, members, offsets):
    assert got["bboxes"].shape[0] == len(groups) > 0
    assert torch.equal(got["bboxes"].cpu(), merged["bboxes"])
    assert torch.equal(got["scores"].cpu(), merged["scores"])
    assert torch.equal(got["labels"].cpu(), merged["labels"])
    assert torch.equal(got["members"], members)
    assert torch.equal(got["member_offsets"], offsets)
    assert torch.equal(got["source"], members[offsets[:-1]])


@pytest.mark.parametrize("metric", ["ios", "iou"])
@pytest.mark.parametrize("thr", [0.3, 0.5])
@pytest.mark.parametrize("n_tiles, hw, full", [(1, (512, 512), False), (12, (1100, 1500), False),
                                               (130, (4000, 6000), True)], ids=["1", "12", "13000_candidates"])
def test_nmm_merge_equals_oracle(n_tiles, hw, full, thr, metric):
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    P, M = 512, 100
    org = slice_origins(hw, P, 0.25)[:n_tiles]
    assert len(org) == n_tiles
    recs = _records(n_tiles, P, M, seed=n_tiles, full=full)
    origins = [org[i:i + 4] for i in range(0, n_tiles, 4)]
    if full:
        assert n_tiles * M > 10000
    got = merge_tile_records(recs, origins, hw, merge_iou_thr=thr, nms_type="greedy_nmm", match_metric=metric)
    merged, groups, members, offsets, _, _ = _oracle_nmm(recs, origins, hw, thr, metric, P)
    _assert_merge_equal(got, merged, groups, members, offsets)
    if metric == "ios" and n_tiles > 1:
        assert members.shape[0] > len(groups)                     # something was merged


def test_nmm_merge_score_thr():
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    P, M, hw = 512, 100, (1100, 1500)
    org = slice_origins(hw, P, 0.25)
    recs = _records(len(org), P, M, seed=5)
    origins = [org[i:i + 4] for i in range(0, len(org), 4)]
    got = merge_tile_records(recs, origins, hw, merge_iou_thr=0.5, score_thr=0.4, nms_type="greedy_nmm")
    _assert_merge_equal(got, *_oracle_nmm(recs, origins, hw, 0.5, "ios", P, score_thr=0.4)[:4])
    assert (got["scores"] >= 0.4).all()


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


def test_nmm_merge_synchronises_once_as_the_hard_merge():
    from rsprompter_b200.large_image import merge_tile_records, slice_origins
    P, M, hw = 512, 100, (1100, 1500)
    org = slice_origins(hw, P, 0.25)
    recs = _records(len(org), P, M, seed=6)
    origins = [org[i:i + 4] for i in range(0, len(org), 4)]
    nmm = _host_syncs(lambda: merge_tile_records(recs, origins, hw, merge_iou_thr=0.5, nms_type="greedy_nmm"))
    hard = _host_syncs(lambda: merge_tile_records(recs, origins, hw, merge_iou_thr=0.5))
    assert nmm == hard


def test_nothing_matches_above_one_and_nmm_is_the_hard_merge():
    from rsprompter_b200.large_image import (encode_kept_masks, encode_merged_masks, merge_tile_records,
                                             slice_origins)
    P, M, hw = 128, 20, (300, 400)
    org = slice_origins(hw, P, 0.25)
    recs = _records(len(org), P, M, seed=7, bits=True)
    origins = [org[i:i + 4] for i in range(0, len(org), 4)]
    for metric in ("ios", "iou"):
        got = merge_tile_records(recs, origins, hw, merge_iou_thr=1.5, nms_type="greedy_nmm", match_metric=metric)
        hard = merge_tile_records(recs, origins, hw, merge_iou_thr=1.5)
        for k in ("bboxes", "scores", "labels", "source"):
            assert torch.equal(got[k], hard[k]), k
        k = hard["source"].shape[0]
        assert torch.equal(got["members"], hard["source"]) and torch.equal(got["member_offsets"], torch.arange(k + 1))
        a = encode_merged_masks(recs, origins, got["members"], got["member_offsets"], hw)
        assert a == encode_kept_masks(recs, origins, hard["source"], hw) and len(a) == k > 0


def test_merged_masks_are_the_or_of_the_members():
    from rsprompter_b200.large_image import encode_merged_masks, merge_tile_records, slice_origins
    from rsprompter_b200.results import mask_to_coco_rle
    P, M, hw = 128, 20, (300, 400)
    org = slice_origins(hw, P, 0.25)
    recs = _records(len(org), P, M, seed=8, bits=True)
    origins = [org[i:i + 4] for i in range(0, len(org), 4)]
    got = merge_tile_records(recs, origins, hw, merge_iou_thr=0.3, nms_type="greedy_nmm")
    merged, groups, members, offsets, tiles, offs = _oracle_nmm(recs, origins, hw, 0.3, "ios", P)
    _assert_merge_equal(got, merged, groups, members, offsets)
    masks = [m for t in tiles for m in t["masks"]]
    tile_of = [i for i, t in enumerate(tiles) for _ in range(t["masks"].shape[0])]
    ref = [mask_to_coco_rle(oracle.union_masks([masks[i] for i in g], [offs[tile_of[i]] for i in g], hw).numpy())
           ["counts"] for g in groups]
    assert any(len(g) > 1 for g in groups)
    assert [m["counts"] for m in encode_merged_masks(recs, origins, got["members"], got["member_offsets"], hw)] == ref


def test_seam_split_object_comes_out_whole():
    """One ellipse across the seam of two overlapping tiles: greedy_nmm gives it whole, nms only the kept fragment."""
    from rsprompter_b200 import _lib
    from rsprompter_b200.large_image import (encode_kept_masks, encode_merged_masks, merge_tile_records,
                                             slice_origins)
    from rsprompter_b200.results import ResultRecord, coco_rle_to_mask
    H, W, P = 128, 224, 128
    org = slice_origins((H, W), P, 0.25)
    assert org == [(0, 0), (96, 0)]
    yy, xx = np.mgrid[0:H, 0:W]
    obj = ((yy - 60) / 30.0) ** 2 + ((xx - 115) / 35.0) ** 2 < 1            # scene x 81 .. 149
    rec = ResultRecord(2, 1, (P, P), device="cuda")
    rows = []
    for b, (x0, y0) in enumerate(org):
        crop = obj[:, x0:x0 + P]
        ys, xs = np.nonzero(crop)
        rows.append([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1, 0.9 - 0.1 * b, 3])
        rec.mask_bits[b, 0].copy_(_lib.pack_mask_bits(torch.from_numpy(crop[None]).cuda())[0])
    rec.rows.copy_(torch.tensor(rows, dtype=torch.float32)[:, None])
    rec.counts.copy_(torch.tensor([1, 1], dtype=torch.int32))
    got = merge_tile_records([rec], [org], (H, W), merge_iou_thr=0.5, nms_type="greedy_nmm")
    assert got["member_offsets"].tolist() == [0, 2]
    assert got["bboxes"].cpu().tolist() == [[81.0, 31.0, 150.0, 90.0]]
    m = encode_merged_masks([rec], [org], got["members"], got["member_offsets"], (H, W))
    assert np.array_equal(coco_rle_to_mask(m[0]), obj)
    hard = merge_tile_records([rec], [org], (H, W), merge_iou_thr=0.25)
    assert hard["source"].tolist() == [[0, 0, 0]]
    frag = np.zeros_like(obj)
    frag[:, :P] = obj[:, :P]
    assert np.array_equal(coco_rle_to_mask(encode_kept_masks([rec], [org], hard["source"], (H, W))[0]), frag)


# ---- end to end ---------------------------------------------------------------------------------------------------
def _reference_nmm(model, scene, ratio, thr, metric, batch_size=8):
    """Tiles cut with torch (NCHW batches), predict_records, host records through the oracle merge, the OR of
    shift_masks and the host RLE."""
    from rsprompter_b200.results import mask_to_coco_rle
    H, W = scene.shape[:2]
    P = model.backbone.vision_encoder.arch.image_size
    org = oracle_li.slice_origins((H, W), P, ratio)
    tiles, offs = [], []
    for i in range(0, len(org), batch_size):
        chunk = org[i:i + batch_size]
        pad = chunk + [chunk[-1]] * (min(batch_size, len(org)) - len(chunk))
        x = torch.stack([torch.from_numpy(scene[y0:y0 + P, x0:x0 + P]).permute(2, 0, 1) for x0, y0 in pad])
        x = x.contiguous().cuda()
        x.rsp_norm = model.data_preprocessor._norm3()
        host = model.predict_records(x).to_host(non_blocking=False)
        torch.cuda.synchronize()
        tiles += host.instances()[:len(chunk)]
        offs += chunk
    return _compose(tiles, offs, (H, W), thr, metric, P)


def _compose(tiles, offs, hw, thr, metric, P):
    from rsprompter_b200.results import mask_to_coco_rle
    boxes_only = [{k: t[k] for k in ("bboxes", "scores", "labels")} for t in tiles]
    merged, groups = oracle.merge_results_by_nmm(boxes_only, offs, hw, thr, metric, patch=P)
    masks = [m[:P, :P] for t in tiles for m in t["masks"]]
    tile_of = [i for i, t in enumerate(tiles) for _ in range(t["masks"].shape[0])]
    rles = [mask_to_coco_rle(oracle.union_masks([masks[i] for i in g], [offs[tile_of[i]] for i in g], hw).numpy())
            ["counts"] for g in groups]
    return merged, rles


def _assert_equal(ds, ref, rles, hw):
    p = ds.pred_instances
    assert len(rles) > 0
    assert torch.equal(p.bboxes.cpu(), ref["bboxes"])
    assert torch.equal(p.scores.cpu(), ref["scores"])
    assert torch.equal(p.labels.cpu(), ref["labels"])
    assert [m["counts"] for m in p.masks] == rles
    assert all(m["size"] == list(hw) for m in p.masks)


@pytest.mark.parametrize("kind", ["anchor", "query", "maskrcnn"])
def test_predict_large_image_nmm_equals_reference_composition(kind):
    from rsprompter_b200.large_image import predict_large_image
    model = _model(kind)
    scene = _scene(1100, 1500, seed=1)
    ds = predict_large_image(model, scene, merge_iou_thr=0.3, merge_nms_type="greedy_nmm")
    ref, rles = _reference_nmm(model, scene, 0.25, 0.3, "ios")
    _assert_equal(ds, ref, rles, (1100, 1500))
    iou = predict_large_image(model, scene, merge_iou_thr=0.5, merge_nms_type="greedy_nmm", merge_match_metric="iou")
    _assert_equal(iou, *_reference_nmm(model, scene, 0.25, 0.5, "iou"), (1100, 1500))


def test_resized_patch_scene():
    from rsprompter_b200.large_image import predict_large_image, run_tiles
    model = _model("query")
    scene = _scene(1100, 1500, seed=1)
    P = 700                                                       # records of 700 x 704: windows on a wider canvas
    ds = predict_large_image(model, scene, patch_size=P, merge_iou_thr=0.3, merge_nms_type="greedy_nmm")
    records, batches = run_tiles(model, scene, patch_size=P)
    tiles, offs = [], []
    for rec, org in zip(records, batches):
        assert rec.hw == (700, 704)
        tiles += rec.to_host(non_blocking=False).instances()[:len(org)]
        offs += org
    _assert_equal(ds, *_compose(tiles, offs, (1100, 1500), 0.3, "ios", P), (1100, 1500))


def test_nmm_cuda_graphs_on_and_off_agree():
    from rsprompter_b200.large_image import predict_large_image
    model = _model("query")
    scene = _scene(700, 1300, seed=4)
    kw = dict(batch_size=4, merge_iou_thr=0.3, merge_nms_type="greedy_nmm")
    off = predict_large_image(model, scene, **kw).pred_instances
    model.enable_cuda_graphs()
    try:
        on = predict_large_image(model, scene, **kw).pred_instances
        again = predict_large_image(model, scene, **kw).pred_instances
    finally:
        model.enable_cuda_graphs(False)
    assert len(off.masks) > 0
    for r in (on, again):
        for k in ("bboxes", "scores", "labels"):
            assert torch.equal(getattr(r, k), getattr(off, k)), k
        assert r.masks == off.masks


def test_nmm_cli_writes_the_result_json(tmp_path):
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
    main([str(cfg), str(img), "--checkpoint", str(ckpt), "--out", str(out), "--merge-nms-type", "greedy_nmm",
          "--merge-match-metric", "iou", "--merge-iou-thr", "0.5"])
    got = json.loads(out.read_text())
    ref = coco_results(predict_large_image(model, scene, merge_iou_thr=0.5, merge_nms_type="greedy_nmm",
                                           merge_match_metric="iou"))
    assert len(ref) > 0 and got == json.loads(json.dumps(ref))
