"""Segment-everything over a whole scene without a GPU: oracle.restate_scene_mask_generation's crop-edge rule and uncrop
pinned to transformers' _is_box_near_crop_edge and _pad_masks; the windows against slice_origins; the merge's tie
order; the arguments generate_scene_masks refuses before any device work; what ptxas made of the crop variant of
rsp_sam_mask_stats."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hf_near(boxes, crop_box, hw):
    from transformers.models.sam.image_processing_sam import _is_box_near_crop_edge
    H, W = hw
    return _is_box_near_crop_edge(boxes, list(crop_box), [0, 0, W, H], atol=20)


def _crafted(crop_box):
    """Boxes in crop pixels whose sides sit 19, 20, 21 and 22 px inside each crop side, on the crop's sides, an empty
    mask's [0, 0, 0, 0], the whole crop, and seeded random boxes."""
    x0, y0, x1, y1 = crop_box
    w, h = x1 - x0, y1 - y0
    rows = [[0, 0, 0, 0], [0, 0, w - 1, h - 1], [0, 0, w, h]]
    for d in (19, 20, 21, 22):
        mid_x, mid_y = w // 2, h // 2
        rows += [[d, mid_y, mid_x, mid_y + 1], [mid_x, d, mid_x + 1, mid_y], [mid_x, mid_y, w - d, mid_y + 1],
                 [mid_x, mid_y, mid_x + 1, h - d]]
    g = torch.Generator().manual_seed(w * 31 + h)
    a = torch.stack([torch.randint(0, w, (64,), generator=g), torch.randint(0, h, (64,), generator=g)], 1)
    b = torch.stack([torch.randint(0, w, (64,), generator=g), torch.randint(0, h, (64,), generator=g)], 1)
    rand = torch.cat([torch.minimum(a, b), torch.maximum(a, b)], 1)
    return torch.cat([torch.tensor(rows, dtype=torch.int64), rand])


# (scene (H, W), patch): six windows with inward-shifted last ones; a scene smaller than the patch (one window that
# is the scene); a scene overhung vertically by every window; a scene just over one patch wide
EDGE_CASES = [((1536, 2048), 1024), ((600, 800), 1024), ((600, 2500), 1024), ((1024, 1030), 1024)]


@pytest.mark.parametrize("hw, patch", EDGE_CASES)
def test_edge_rule_matches_hf(hw, patch):
    from oracle import restate_scene_mask_generation as O
    crops = O.crop_boxes(hw, patch, 0.25)
    flagged = 0
    for cb in crops:
        boxes = _crafted(cb)
        got = O.near_crop_edge(boxes, cb, hw)
        assert torch.equal(got, _hf_near(boxes, cb, hw)), cb
        flagged += int(got.sum())
    if len(crops) == 1:
        assert flagged == 0                       # the crop box is the scene: the rule is a no-op
    else:
        assert flagged > 0


def test_edge_rule_worked_examples():
    """The middle top window of a 1536 x 2048 scene at P = 1024: its left and right sides (x = 768, 1792) and its
    bottom (y = 1024) are interior, its top is the scene's."""
    from oracle import restate_scene_mask_generation as O
    hw, cb = (1536, 2048), (768, 0, 1792, 1024)
    boxes = torch.tensor([[20, 300, 500, 400],     # 20 px from the left side: near
                          [21, 300, 500, 400],     # 21 px: not
                          [300, 300, 1004, 400],   # right side 1772, 20 px from 1792: near
                          [300, 300, 1003, 400],   # 21 px: not
                          [300, 0, 500, 400],      # on the top side, which is the scene's: not
                          [300, 300, 500, 1004],   # bottom 20 px from the interior bottom side: near
                          [0, 0, 0, 0]])           # an empty mask: its left side is on the crop's left side: near
    expect = torch.tensor([True, False, True, False, False, True, True])
    assert torch.equal(O.near_crop_edge(boxes, cb, hw), expect)
    assert torch.equal(_hf_near(boxes, cb, hw), expect)
    # the inward-shifted last window (1024, 512, 2048, 1536): right and bottom are the scene's, left and top interior
    cb = (1024, 512, 2048, 1536)
    boxes = torch.tensor([[500, 500, 1023, 1023], [500, 500, 1003, 1003], [0, 500, 10, 600], [500, 20, 600, 30],
                          [500, 21, 600, 30]])
    expect = torch.tensor([False, False, True, True, False])
    assert torch.equal(O.near_crop_edge(boxes, cb, hw), expect)
    assert torch.equal(_hf_near(boxes, cb, hw), expect)


@pytest.mark.parametrize("hw, patch", EDGE_CASES)
def test_uncrop_matches_hf_pad_masks(hw, patch):
    from transformers.models.sam.image_processing_sam import _pad_masks

    from oracle import restate_scene_mask_generation as O
    g = torch.Generator().manual_seed(hw[0] + hw[1])
    for cb in O.crop_boxes(hw, patch, 0.25):
        m = torch.rand(2, cb[3] - cb[1], cb[2] - cb[0], generator=g) > 0.5
        assert torch.equal(O.uncrop(m, cb, hw), _pad_masks(m, list(cb), hw[0], hw[1]))


@pytest.mark.parametrize("hw, patch, ratio", [((1536, 2048), 1024, 0.25), ((600, 800), 1024, 0.25),
                                              ((600, 2500), 1024, 0.25), ((4096, 4096), 1024, 0.25),
                                              ((3000, 2000), 512, 0.5), ((1000, 1000), 300, 0.0)])
def test_windows_are_slice_origins_cut_to_the_scene(hw, patch, ratio):
    from oracle import restate_large_image as L
    from oracle import restate_scene_mask_generation as O
    from rsprompter_b200 import mask_generation as mg
    from rsprompter_b200.large_image import slice_origins
    got = mg.scene_crop_boxes(hw, patch, ratio)
    H, W = hw
    assert got == O.crop_boxes(hw, patch, ratio)
    assert [(x0, y0) for x0, y0, _, _ in got] == slice_origins(hw, patch, ratio) == L.slice_origins(hw, patch, ratio)
    for x0, y0, x1, y1 in got:
        assert x1 == min(x0 + patch, W) and y1 == min(y0 + patch, H) and x1 > x0 and y1 > y0


def test_windows_of_a_six_window_scene():
    from rsprompter_b200 import mask_generation as mg
    assert mg.scene_crop_boxes((1536, 2048), 1024, 0.25) == [
        (0, 0, 1024, 1024), (768, 0, 1792, 1024), (1024, 0, 2048, 1024),
        (0, 512, 1024, 1536), (768, 512, 1792, 1536), (1024, 512, 2048, 1536)]


def test_merge_breaks_score_ties_by_window_then_rank():
    """Equal scores everywhere and boxes that do not overlap: the keep order is (window, rank in the window); one box
    of window 1 overlapping window 0's first box is suppressed by it, whatever its rank."""
    from oracle import restate_scene_mask_generation as O
    crops = [(0, 0, 100, 100), (80, 0, 180, 100)]
    win0 = dict(index=torch.tensor([5, 2]), scores=torch.tensor([0.5, 0.5]), stability=torch.tensor([1.0, 1.0]),
                boxes=torch.tensor([[0, 0, 10, 10], [30, 30, 40, 40]]))
    win1 = dict(index=torch.tensor([7, 1, 4]), scores=torch.tensor([0.5, 0.5, 0.5]),
                stability=torch.tensor([1.0, 1.0, 1.0]),
                boxes=torch.tensor([[-80, 0, -70, 10], [50, 50, 60, 60], [70, 70, 80, 80]]))
    pts = [torch.zeros(4, 2), torch.zeros(4, 2)]
    m = O.merge([win0, win1], crops, pts, 0.7)
    assert m["tiles"].tolist() == [0, 0, 1, 1]
    assert m["candidates"].tolist() == [5, 2, 1, 4]
    assert m["rank"].tolist() == [0, 1, 1, 2]
    assert m["boxes"].tolist() == [[0, 0, 10, 10], [30, 30, 40, 40], [130, 50, 140, 60], [150, 70, 160, 80]]
    # a higher score goes first whatever its window
    win1["scores"] = torch.tensor([0.5, 0.5, 0.9])
    m = O.merge([win0, win1], crops, pts, 0.7)
    assert m["candidates"].tolist() == [4, 5, 2, 1]


@pytest.mark.parametrize("kw, msg", [
    (dict(crops_n_layers=1), "stack expects each tensor to be equal size"),
    (dict(max_hole_area=10.0), "max_hole_area"),
    (dict(points_per_batch=0), "points_per_batch"),
    (dict(points_per_side=0), "points_per_side"),
    (dict(patch_size=0), "patch_size"),
    (dict(overlap_ratio=1.0), "overlap_ratio"),
    (dict(overlap_ratio=-0.1), "overlap_ratio"),
    (dict(batch_size=0), "batch_size"),
    (dict(min_mask_region_area=float("nan")), "min_mask_region_area"),
])
def test_arguments_are_refused_before_device_work(kw, msg):
    from rsprompter_b200.mask_generation import generate_scene_masks
    # no model: the parameters and the scene are checked before it is looked at
    with pytest.raises(ValueError, match=msg):
        generate_scene_masks(None, torch.zeros(3, 64, 64, dtype=torch.uint8), **kw)


@pytest.mark.parametrize("scene", [torch.zeros(3, 64, 64), torch.zeros(64, 64, 3, dtype=torch.uint8),
                                   torch.zeros(1, 3, 64, 64, dtype=torch.uint8), None])
def test_scenes_that_are_not_uint8_chw_are_refused(scene):
    from rsprompter_b200.mask_generation import generate_scene_masks
    with pytest.raises(ValueError, match="uint8 RGB tensor"):
        generate_scene_masks(None, scene)


def test_crop_stats_kernel_does_not_spill():
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
        if m and cur is not None and "crop_mask_stats_finish" in cur:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 1, sorted(found)
    assert all(v == (0, 0) for v in found.values()), found
