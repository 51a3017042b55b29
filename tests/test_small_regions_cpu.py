"""SAM's small-region removal without a GPU: oracle.restate_small_regions on hand-worked cases; the label order of
cv2.connectedComponentsWithStats that the GPU kernel's islands fallback follows (2 x 2 pixel blocks in raster order,
not pixels); generate_masks refusing a non-finite min_mask_region_area before any device work; what ptxas made of the
rsp_mask_small_regions_bits kernels."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rsr(mask, area, mode):
    from oracle.restate_small_regions import remove_small_regions
    out, changed = remove_small_regions(np.asarray(mask, dtype=bool), area, mode)
    return np.asarray(out, dtype=bool), changed


@pytest.mark.parametrize("area, filled", [(5, True), (4.5, True), (4, False)])
def test_hole_below_the_area_is_filled_and_one_at_it_is_not(area, filled):
    m = np.ones((10, 10), bool)
    m[4:6, 4:6] = False                                           # a hole of 4 pixels
    out, changed = _rsr(m, area, "holes")
    assert changed == filled
    assert (out == (np.ones_like(m) if filled else m)).all()


def test_small_border_background_region_is_filled():
    m = np.ones((6, 7), bool)
    m[0, 0] = m[0, 1] = False                                     # background touching the border
    m[5, 6] = False
    out, changed = _rsr(m, 3, "holes")
    assert changed and out.all()


def test_diagonal_contacts_connect():
    m = np.zeros((5, 5), bool)
    for i in range(4):
        m[i, i] = True                                            # one 8-connected island of 4 (four 4-connected ones)
    out, changed = _rsr(m, 4, "islands")
    assert not changed and (out == m).all()
    out, changed = _rsr(m, 5, "islands")
    assert changed and (out == m).all()                           # all small: the largest, i.e. all of it, stays
    # background: the diagonal of background pixels is one component of 4 pixels
    out, changed = _rsr(~m, 5, "holes")
    assert changed and out.all()


def test_single_small_island_is_unchanged_but_counts_as_changed():
    m = np.zeros((8, 8), bool)
    m[3, 3] = True
    out, changed = _rsr(m, 5, "islands")
    assert changed and (out == m).all()


def test_equal_largest_islands_keep_the_first_cv2_label():
    """Two islands of one pixel, both small: the one cv2 labels first is the one whose 2 x 2 block comes first,
    (row 1, col 10) before (row 0, col 20), though (0, 20) comes first in pixel raster order."""
    m = np.zeros((4, 32), bool)
    m[1, 10] = m[0, 20] = True
    out, changed = _rsr(m, 2, "islands")
    assert changed
    expect = np.zeros_like(m)
    expect[1, 10] = True
    assert (out == expect).all()


def test_filled_hole_joins_two_islands():
    """A background column between two islands of 6 is a hole of 3: filled first, it makes one island of 15 >= 7
    that stays whole, where islands alone would keep only one of the two."""
    from oracle.restate_small_regions import postprocess_small_regions
    import torch
    m = np.ones((3, 5), bool)
    m[:, 2] = False
    h, ch = _rsr(m, 7, "holes")
    assert ch and h.all()
    i, ch = _rsr(h, 7, "islands")
    assert not ch and i.all()
    alone, ch = _rsr(m, 7, "islands")
    assert ch and alone.sum() == 6
    pp = postprocess_small_regions(torch.from_numpy(m)[None], 7, 0.7)
    assert pp["changed"].tolist() == [True] and pp["masks"][0].all() and pp["boxes"].tolist() == [[0, 0, 4, 2]]


def test_second_nms_ranks_unchanged_masks_first_and_keeps_ties_in_order():
    import torch

    from oracle.restate_small_regions import postprocess_small_regions
    masks = torch.zeros(4, 20, 20, dtype=torch.bool)
    masks[0, 0:4, 0:4] = True
    masks[0, 15, 15] = True                                       # an island of 1: changed
    masks[1, 10:14, 0:4] = True                                   # clean
    masks[2, 0:4, 10:14] = True
    masks[2, 1, 11] = False                                       # a hole of 1: changed
    masks[3, 15:19, 5:9] = True                                   # clean
    pp = postprocess_small_regions(masks, 2, 0.7)
    assert pp["index"].tolist() == [1, 3, 0, 2]
    assert pp["changed"].tolist() == [True, False, True, False]
    assert pp["boxes"].tolist() == [[0, 10, 3, 13], [5, 15, 8, 18], [0, 0, 3, 3], [10, 0, 13, 3]]


def _first_block_order(labels, n):
    from scipy import ndimage
    H, W = labels.shape
    ys, xs = np.indices((H, W))
    block = (ys // 2) * ((W + 1) // 2) + xs // 2
    pixel = ys * W + xs
    idx = np.arange(1, n)
    return (np.asarray(ndimage.minimum(block, labels, idx)), np.asarray(ndimage.minimum(pixel, labels, idx)))


@pytest.mark.parametrize("hw, threads", [((64, 96), 1), ((2000, 2000), 8), ((1999, 2001), 8)])
def test_cv2_numbers_components_by_first_2x2_block(hw, threads):
    """The islands fallback's tie-break: cv2 (default algorithm, 8-connectivity) numbers components in raster order
    of the first 2 x 2 pixel block (y // 2, x // 2) each touches, also on large images labelled by several threads;
    the pixel raster order differs on the same image."""
    import cv2
    rng = np.random.default_rng(hw[0] + threads)
    m = (rng.random(hw) < 0.35).astype(np.uint8)
    prev = cv2.getNumThreads()
    cv2.setNumThreads(threads)
    try:
        n, labels, _, _ = cv2.connectedComponentsWithStats(m, 8)
    finally:
        cv2.setNumThreads(prev)
    assert n > 100
    block, pixel = _first_block_order(labels, n)
    assert (np.diff(block) > 0).all()
    assert not (np.diff(pixel) > 0).all()


@pytest.mark.parametrize("area", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_area_is_refused_before_device_work(area):
    from rsprompter_b200.mask_generation import generate_masks
    with pytest.raises(ValueError, match="min_mask_region_area"):
        generate_masks(None, None, min_mask_region_area=area)


def test_small_regions_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "regions.ptxas.log")) as f:
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
        if m and cur is not None and "regions_" in cur:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 7, sorted(found)
    assert all(v == (0, 0) for v in found.values()), found
