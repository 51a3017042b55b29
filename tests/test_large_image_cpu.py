"""Large-scene inference without a GPU: the slicing rule against worked examples of sahi's slice_image windows, the
oracle merge on hand-built tiles, the argument checks of the placed RLE entry points (they run before any launch),
and that no placed RLE kernel spills."""
import ctypes
import os
import re
import sys

import pytest
import torch

from oracle import restate_large_image as oracle
from rsprompter_b200 import _lib
from rsprompter_b200.large_image import slice_origins

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _grid(xs, ys):
    return [(x, y) for y in ys for x in xs]


@pytest.mark.parametrize("hw, ratio, xs, ys", [
    ((2000, 3000), 0.25, [0, 768, 1536, 1976], [0, 768, 976]),
    ((1024, 1024), 0.25, [0], [0]),                              # exact fit: one tile
    ((1024, 1792), 0.25, [0, 768], [0]),                         # exact fit of two overlapping tiles
    ((800, 3000), 0.25, [0, 768, 1536, 1976], [0]),              # shorter than the patch: tiles overhang
    ((2000, 3000), 0.2, [0, 820, 1640, 1976], [0, 820, 976]),    # overlap int(204.8) = 204
    ((2000, 3000), 0.0, [0, 1024, 1976], [0, 976]),
])
def test_slice_origins_worked_examples(hw, ratio, xs, ys):
    got = slice_origins(hw, 1024, ratio)
    assert got == _grid(xs, ys)
    assert got == oracle.slice_origins(hw, 1024, ratio)


def test_slice_origins_cover_the_scene():
    for hw in [(1, 1), (513, 4097), (5000, 7001), (1024, 1025)]:
        for ratio in (0.0, 0.1, 0.25, 0.5):
            org = slice_origins(hw, 512, ratio)
            assert org == oracle.slice_origins(hw, 512, ratio)
            cover = torch.zeros(hw, dtype=torch.bool)
            for x0, y0 in org:
                assert 0 <= x0 and 0 <= y0 and (x0 + 512 <= hw[1] or x0 == 0) and (y0 + 512 <= hw[0] or y0 == 0)
                cover[y0:y0 + 512, x0:x0 + 512] = True
            assert bool(cover.all())


def _tile(boxes, scores, labels):
    return dict(bboxes=torch.tensor(boxes, dtype=torch.float32), scores=torch.tensor(scores),
                labels=torch.tensor(labels))


def test_oracle_merge_hand_built():
    # tile 0 at (0, 0), tile 1 at (768, 0): the object at scene x 800..900 is seen by both
    t0 = _tile([[800, 10, 900, 60], [10, 10, 50, 50], [800, 10, 900, 60]], [0.9, 0.5, 0.4], [1, 2, 3])
    t1 = _tile([[32, 10, 132, 60], [32, 12, 132, 61], [300, 300, 310, 310]], [0.8, 0.95, 0.3], [1, 1, 1])
    merged, keep = oracle.merge_results_by_nms([t0, t1], [(0, 0), (768, 0)], (1024, 2048), 0.25)
    # the duplicate of label 1 goes (0.95 keeps, 0.9 and 0.8 are suppressed); label 3 at the same place stays
    assert keep.tolist() == [4, 1, 2, 5]
    assert merged["scores"].tolist() == sorted(merged["scores"].tolist(), reverse=True)
    assert merged["labels"].tolist() == [1, 2, 3, 1]
    assert merged["bboxes"][0].tolist() == [800.0, 12.0, 900.0, 61.0]


def test_oracle_clip_to_tile_window():
    t = _tile([[-5, 900, 200, 1100]], [0.5], [0])
    inst = oracle.shift_predictions([t], [(100, 0)], (800, 3000), patch=1024)
    assert inst["bboxes"].tolist() == [[100.0, 800.0, 300.0, 800.0]]


def _placed_status(fields, packed=1):
    desc = (ctypes.c_int64 * 18)(0, 128, 1024, 1024, 1024, 2000, 3000, 0, 0, *fields)   # mask 0 valid, mask 1 not
    fake = ctypes.c_void_p(16)                                    # never dereferenced: the checks precede every launch
    return _lib._lib.rsp_mask_rle_placed_lengths(fake, packed, fake, ctypes.cast(desc, ctypes.c_void_p), 2, fake, None)


@pytest.mark.parametrize("fields", [
    (0, 2500, 1024, 1024, 1024, 50000, 50000, 0, 0),         # canvas above 2^31 - 1 pixels
    (0, 128, 1024, 1024, 1024, 0, 3000, 0, 0),               # empty canvas
    (0, 128, 1024, 1024, 1024, 2000, 3000, 2000, 0),         # origin below the canvas
    (0, 128, 1024, 1024, 1024, 2000, 3000, 0, -1),           # origin left of the canvas
    (0, 128, 1024, 1024, 1024, 2000, 3000, 1000, 0),         # visible rows leave the canvas
    (0, 128, 1024, 1025, 1000, 4000, 3000, 0, 0),            # more visible rows than the source has
    (0, 128, 1024, 1000, 1025, 4000, 3000, 0, 0),            # more visible columns than a source row holds
    (0, 128, 1024, 0, 1000, 4000, 3000, 0, 0),               # empty visible extent
    (-1, 128, 1024, 1000, 1000, 4000, 3000, 0, 0),           # negative offset
])
def test_mask_rle_placed_rejects_bad_descriptors(fields):
    assert _placed_status(fields) == 1
    assert b"mask 1" in _lib._lib.rsp_last_error()


def test_mask_rle_placed_bool_source_width():
    # a bool source row of 128 bytes holds 128 pixels, a packed one 1024
    assert _placed_status((0, 128, 1024, 100, 129, 4000, 3000, 0, 0), packed=0) == 1


def test_placed_symbols_in_header_and_binding():
    with open(os.path.join(ROOT, "include", "rsp_b200.h")) as f:
        header = f.read()
    for name in ("rsp_mask_rle_placed_lengths", "rsp_mask_rle_placed_write"):
        assert re.search(rf"\bint {name}\(", header)
        assert name in _lib.declared_symbols()


def test_detectors_without_tile_records_are_refused():
    from rsprompter_b200.detectors import SAMSegMask2Former
    from rsprompter_b200.large_image import predict_large_image
    with pytest.raises(NotImplementedError, match="SAMSegMask2Former"):
        predict_large_image(SAMSegMask2Former.__new__(SAMSegMask2Former), None)


def test_rle_kernels_do_not_spill():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "rle.ptxas.log")) as f:
        log = f.read()
    spills = {}
    for name, st, ld in re.findall(r"Function properties for (\S*mask_rle_kernel\S*)\s+\d+ bytes stack frame, "
                                   r"(\d+) bytes spill stores, (\d+) bytes spill loads", log):
        spills[re.search(r"mask_rle_kernelI(\w+)EE", name).group(1)] = (int(st), int(ld))
    assert len(spills) == 8, sorted(spills)                       # packed x write x placed
    assert all(v == (0, 0) for v in spills.values()), spills
