"""SAM mask generation without a GPU: oracle.restate_mask_generation pinned to transformers' own point grid,
normalisation, post_process_masks(binarize=False), filter_masks and post_process_for_mask_generation; the generator's
own point grid; the arguments generate_masks refuses before any device work; what ptxas made of rsp_sam_mask_stats."""
import os
import re
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1024, 1024), (600, 800), (800, 600), (333, 517)]


@pytest.mark.parametrize("n", [1, 5, 32])
@pytest.mark.parametrize("hw", SIZES)
def test_point_grid_matches_hf(hw, n):
    from transformers.models.sam.image_processing_sam import _build_point_grid, _normalize_coordinates

    from oracle import restate_mask_generation as R
    from rsprompter_b200 import mask_generation as mg
    grid = _build_point_grid(n)
    assert torch.equal(R.build_point_grid(n), grid)
    pts = grid * torch.tensor(hw).flip(dims=(0,)).unsqueeze(0)         # _generate_crop_images, the whole-image crop
    ref = _normalize_coordinates(1024, pts, hw)
    o_pts, o_model = R.grid_prompts(n, hw)
    g_pts, g_model = mg.point_grid(n, hw, 1024)
    for a, b in ((o_pts, pts), (g_pts, pts), (o_model, ref), (g_model, ref)):
        assert a.dtype == b.dtype == torch.float32 and torch.equal(a, b)


def _decoder_outputs(pb: int, seed: int):
    """Low-res logits with region structure (a smooth field plus a little noise, so boxes differ and overlap) and
    tie-free iou scores."""
    g = torch.Generator().manual_seed(seed)
    field = F.interpolate(torch.randn(pb, 3, 6, 6, generator=g) * 8, (256, 256), mode="bilinear", align_corners=False)
    low = field + 1e-2 * torch.randn(pb, 3, 256, 256, generator=g)
    iou = torch.rand(pb, 3, generator=g)
    return low, iou


def _between(values: torch.Tensor, q: float) -> float:
    """A threshold strictly between two neighbouring distinct finite values near quantile q."""
    v = torch.unique(values[torch.isfinite(values)].double())
    i = max(1, min(len(v) - 1, int(q * len(v))))
    return float((v[i - 1] + v[i]) / 2)


@pytest.mark.parametrize("hw", SIZES)
def test_restatement_matches_hf_pipeline(hw):
    from transformers import SamImageProcessor

    from oracle import restate_mask_generation as R
    proc = SamImageProcessor()
    H, W = hw
    reshaped = proc._get_preprocess_shape(hw, 1024)
    low, iou = _decoder_outputs(16, seed=H * 7 + W)
    stats = R.mask_stats(R.upscale(low, hw, reshaped).flatten(0, 1), 0.0, 1.0)
    pred_thr = _between(iou.flatten(), 0.3)
    passed = iou.flatten() > pred_thr
    stab_thr = _between(stats["stability"][passed], 0.3)
    kw = dict(pred_iou_thresh=pred_thr, stability_score_thresh=stab_thr, stability_score_offset=1.0, mask_threshold=0.0)

    # HF: MaskGenerationPipeline._forward (one point batch) + postprocess
    masks = proc.post_process_masks([low], [hw], [reshaped], mask_threshold=0.0, binarize=False)[0]
    rle, scores, boxes = proc.filter_masks(masks, iou, hw, [0, 0, W, H], kw["pred_iou_thresh"],
                                           kw["stability_score_thresh"], kw["mask_threshold"],
                                           kw["stability_score_offset"])
    hf_masks, hf_scores, _, hf_boxes = proc.post_process_for_mask_generation(rle, scores, boxes, 0.7)

    got = R.generate(low, iou, hw, reshaped, crops_nms_thresh=0.7, **kw)
    assert 0 < got["after_iou"] < got["candidates"]
    assert 0 < got["after_stability"] < got["after_iou"]
    assert 0 < got["after_nms"] < got["after_stability"]
    assert torch.equal(got["scores"], hf_scores)
    assert torch.equal(got["boxes"], hf_boxes)
    assert torch.equal(got["masks"], torch.stack(hf_masks))
    assert torch.equal(iou.flatten()[got["index"]], hf_scores)


def test_disabled_thresholds_keep_every_candidate():
    from oracle import restate_mask_generation as R
    low, iou = _decoder_outputs(4, seed=3)
    got = R.generate(low, iou, (600, 800), (768, 1024), pred_iou_thresh=0.0, stability_score_thresh=0.0,
                     crops_nms_thresh=1.0)
    assert got["after_iou"] == got["after_stability"] == got["candidates"] == 12
    assert torch.equal(got["index"], torch.sort(iou.flatten(), descending=True, stable=True).indices)


@pytest.mark.parametrize("kw, msg", [
    (dict(crops_n_layers=1), "crops_n_layers"),
    (dict(max_hole_area=10.0), "max_hole_area"),
    (dict(max_sprinkle_area=10.0), "max_sprinkle_area"),
    (dict(points_per_batch=0), "points_per_batch"),
    (dict(points_per_batch=-3), "points_per_batch"),
    (dict(points_per_side=0), "points_per_side"),
])
def test_arguments_are_refused_before_device_work(kw, msg):
    from rsprompter_b200.mask_generation import generate_masks
    # no model and no image: the parameters are checked before either is looked at
    with pytest.raises(ValueError, match=msg):
        generate_masks(None, None, **kw)


def test_crop_layer_error_says_why():
    from rsprompter_b200.mask_generation import generate_masks
    with pytest.raises(ValueError, match="stack expects each tensor to be equal size"):
        generate_masks(None, None, crops_n_layers=2)


def test_sam_mask_stats_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "detect.ptxas.log")) as f:
        log = f.read()
    entry = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
    spills = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    found, cur = {}, None
    for line in log.splitlines():
        m = entry.search(line)
        if m:
            cur = m.group(1)
            continue
        m = spills.search(line)
        if m and cur is not None and "sam_mask_stats" in cur:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 2, sorted(found)
    assert all(v == (0, 0) for v in found.values()), found
