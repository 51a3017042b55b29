"""Coarse layers of segment-everything over a whole scene, without a GPU: oracle.restate_scene_layers' antialiased
resize against torchvision's, the host weight tables of rsp_resize_aa_pad_u8 against the oracle, the windows of each
layer, the geometric guarantee per layer, the cross-layer merge, argument refusals and the spill check."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SIZE_PAIRS = [((2048, 1500), (1024, 750)), ((1500, 900), (1024, 614)), ((600, 800), (768, 1024)),
              ((1037, 2311), (460, 1024)), ((333, 517), (1024, 1024)),
              ((500, 700), (500, 350)), ((640, 300), (200, 300)), ((97, 131), (97, 131))]


@pytest.mark.parametrize("src, dst", SIZE_PAIRS)
def test_oracle_resize_is_torchvision_antialiased_uint8(src, dst):
    from torchvision.transforms.v2 import functional as tvF

    from oracle import restate_scene_layers as O
    img = torch.from_numpy(np.random.default_rng(sum(src)).integers(0, 256, (3, *src), dtype=np.uint8))
    ref = tvF.resize(img, list(dst), interpolation=tvF.InterpolationMode.BILINEAR, antialias=True)
    assert np.array_equal(O.resize_aa(img.numpy(), dst), ref.numpy())


@pytest.mark.parametrize("n_in, n_out", [(2048, 1024), (1500, 1024), (900, 614), (800, 1024), (2311, 1024),
                                         (333, 1024), (8192, 1024), (20000, 1024), (12000, 614), (1024, 1023)])
def test_weight_tables_are_the_oracle_weights(n_in, n_out):
    from oracle import restate_scene_layers as O
    from rsprompter_b200 import _lib
    tab, prec = _lib.resize_aa_table(n_in, n_out)
    xmin, xsize, wi, oprec = O.aa_weights(n_in, n_out)
    assert prec == oprec and tab.dtype == torch.int32
    assert np.array_equal(tab[:, 0].numpy(), xmin) and np.array_equal(tab[:, 1].numpy(), xsize)
    assert np.array_equal(tab[:, 2:].numpy().astype(np.int64), wi)


def test_identity_table_is_exact():
    from rsprompter_b200 import _lib
    tab, prec = _lib.resize_aa_table(37, 37)
    assert tab[:, 0].tolist() == list(range(37)) and tab[:, 1].eq(1).all() and tab[:, 2].eq(1 << prec).all()
    p = torch.arange(256)
    assert torch.equal(((1 << (prec - 1)) + p * (1 << prec)) >> prec, p)


@pytest.mark.parametrize("hw", [(1536, 2048), (5000, 3000), (8192, 8192), (900, 20000)])
@pytest.mark.parametrize("coarse", [(2048,), (2048, 4096), (1600, 8192, 30000)])
def test_layer_windows_are_scene_crop_boxes_per_size(hw, coarse):
    from oracle import restate_scene_layers as O
    from rsprompter_b200.mask_generation import scene_crop_boxes, scene_layer_windows
    layers = scene_layer_windows(hw, 1024, 0.25, coarse)
    assert layers == O.layer_windows(hw, 1024, 0.25, coarse)
    assert layers[0] == (0, scene_crop_boxes(hw, 1024, 0.25))
    for (l, boxes), (_, prev) in zip(layers[1:], layers):
        assert boxes == scene_crop_boxes(hw, coarse[l - 1], 0.25) and boxes != prev
    covering = [l for l, c in enumerate(coarse, 1) if c >= max(hw)]
    if covering:                       # the first size that covers the scene is one window; later ones run not at all
        assert (covering[0], [(0, 0, hw[1], hw[0])]) in layers
        assert not any(l in covering[1:] for l, _ in layers)


def test_a_base_layer_that_is_the_scene_takes_no_coarse_layer():
    from rsprompter_b200.mask_generation import scene_layer_windows
    assert scene_layer_windows((600, 1000), 1024, 0.25, (2048, 4096)) == [(0, [(0, 0, 1000, 600)])]


@pytest.mark.parametrize("P, ratio", [(2048, 0.25), (4096, 0.25), (3000, 0.2)])
def test_every_small_box_lies_inside_some_window_of_its_layer(P, ratio):
    """A box of extent below int(overlap_ratio * P) - 42 lies more than 20 px inside the interior edges of some window
    of that layer, so the crop-edge rule keeps it there."""
    from rsprompter_b200.mask_generation import scene_crop_boxes
    hw = (9000, 11000)
    crops = scene_crop_boxes(hw, P, ratio)
    ext = int(ratio * P) - 43
    g = torch.Generator().manual_seed(P)
    for _ in range(400):
        bw, bh = (torch.randint(1, ext + 1, (2,), generator=g)).tolist()
        x0 = int(torch.randint(0, hw[1] - bw, (1,), generator=g))
        y0 = int(torch.randint(0, hw[0] - bh, (1,), generator=g))
        x1, y1 = x0 + bw, y0 + bh

        def inside(c):
            cx0, cy0, cx1, cy1 = c
            return ((cx0 == 0 or x0 - cx0 > 20) and (cy0 == 0 or y0 - cy0 > 20)
                    and (cx1 == hw[1] or cx1 - x1 > 20) and (cy1 == hw[0] or cy1 - y1 > 20)
                    and cx0 <= x0 and cy0 <= y0 and x1 <= cx1 and y1 <= cy1)
        assert any(inside(c) for c in crops), (x0, y0, x1, y1)


def _rows(boxes, layer):
    n = len(boxes)
    return dict(boxes=torch.tensor(boxes, dtype=torch.int64), scores=torch.rand(n), tiles=torch.zeros(n, dtype=torch.int64))


def test_cross_layer_merge_worked_examples():
    from oracle import restate_scene_layers as O
    base = _rows([[0, 0, 100, 100], [500, 500, 520, 520], [505, 505, 525, 525]], 0)   # base rows overlap each other
    coarse = _rows([[2, 2, 101, 99],              # overlaps base row 0: dropped
                    [1000, 1000, 1800, 1700],     # overlaps nothing: kept
                    [1010, 1000, 1800, 1700],     # overlaps the coarse row kept before it: dropped
                    [0, 0, 400, 400]], 1)         # IoU with base row 0 is 1/16: kept
    whole = _rows([[1000, 1000, 1800, 1690], [3000, 0, 3100, 50]], 2)
    m = O.merge_layers([(0, base), (1, coarse), (2, whole)], 0.5)
    assert m["layers"].tolist() == [0, 0, 0, 1, 1, 2]
    assert m["boxes"].tolist() == [[0, 0, 100, 100], [500, 500, 520, 520], [505, 505, 525, 525],
                                   [1000, 1000, 1800, 1700], [0, 0, 400, 400], [3000, 0, 3100, 50]]


def test_every_base_row_is_kept():
    """Base rows are survivors of the base layer's NMS, which never suppress each other."""
    from oracle import restate_mask_generation as R
    from oracle import restate_scene_layers as O
    g = torch.Generator().manual_seed(3)

    def rand_rows(n):
        xy = torch.randint(0, 2000, (n, 2), generator=g)
        wh = torch.randint(1, 600, (n, 2), generator=g)
        return dict(boxes=torch.cat([xy, xy + wh], 1), scores=torch.rand(n, generator=g))
    base = rand_rows(60)
    keep = R.nms(base["boxes"], base["scores"], 0.5)                  # survivors of the base layer's merge
    base = {k: v[keep] for k, v in base.items()}
    m = O.merge_layers([(0, base), (1, rand_rows(40)), (2, rand_rows(10))], 0.5)
    assert torch.equal(m["boxes"][m["layers"] == 0], base["boxes"])
    assert 0 < int((m["layers"] > 0).sum()) < 50


@pytest.mark.parametrize("kw, msg", [
    (dict(coarse_patch_sizes=(2048, 2048)), "strictly increasing"),
    (dict(coarse_patch_sizes=(4096, 2048)), "strictly increasing"),
    (dict(coarse_patch_sizes=(1024,)), "greater than the patch size 1024"),
    (dict(coarse_patch_sizes=(512, 2048)), "greater than the patch size 1024"),
    (dict(coarse_patch_sizes=(2048.0,)), "integers"),
    (dict(coarse_patch_sizes=(True,)), "integers"),
])
def test_coarse_sizes_are_refused_before_device_work(kw, msg):
    from rsprompter_b200.mask_generation import generate_scene_masks
    # no model: the sizes are checked before it is looked at
    with pytest.raises(ValueError, match=msg):
        generate_scene_masks(None, torch.zeros(3, 64, 64, dtype=torch.uint8), patch_size=1024, **kw)


def test_a_whole_scene_window_of_2_31_pixels_is_refused():
    from rsprompter_b200.mask_generation import generate_scene_masks
    scene = torch.zeros(3, 1, 1, dtype=torch.uint8).expand(3, 40000, 60000)        # a view: no memory
    with pytest.raises(ValueError, match="2\\^31 pixels"):
        generate_scene_masks(None, scene, patch_size=1024, coarse_patch_sizes=(60000,))
    with pytest.raises(TypeError):                              # a smaller coarse window passes on to the model
        generate_scene_masks(None, scene, patch_size=1024, coarse_patch_sizes=(8192,))


def test_resize_aa_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "records.ptxas.log")) as f:
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
        if m and cur is not None and "resize_aa" in cur:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(found) == 2, sorted(found)
    assert all(v == (0, 0) for v in found.values()), found
