"""The folded entry points take their options as arguments (a NULL pointer or a zero size selects the plain form), so
they can express combinations that no operation supports.  Those are rejected before any launch, so the checks hold
without a GPU: fake device pointers are never dereferenced."""
import pytest

from rsprompter_b200 import _lib

P = 1 << 24                    # a fake, 16-byte aligned device pointer
HM = WM = 16                   # low-res maps; the x4 path writes 64 x 64
GEO2 = (256, 256, 200, 240)    # Hb, Wb, crop_h, crop_w: two resizes
GEO1 = (0, 0, 0, 0)            # Hb = 0: one resize


def _status(fn, *args):
    return getattr(_lib._lib, fn)(*args, None), (_lib._lib.rsp_last_error() or b"").decode()


@pytest.mark.parametrize("geo, out_hw, slot, packed, mode, what", [
    (GEO1, (48, 64), (48, 64), 1, 1, "x4"),        # bits after one resize that is not x4
    (GEO1, (64, 64), (80, 64), 1, 2, "x4"),        # x4 bits into larger slots
    (GEO1, (64, 64), (64, 64), 1, 0, "x4"),        # mode 0 with bits
    (GEO2, (150, 200), (150, 200), 0, 0, "mode"),  # mode 0 with two resizes
    (GEO2, (150, 200), (160, 208), 1, 0, "mode"),  # mode 0 with two resizes into bits
    (GEO1, (64, 64), (64, 80), 0, 1, "(Hr, Wr)"),  # bytes whose slot is not the mask
])
def test_mask_paste_rejects_unsupported_combinations(geo, out_hw, slot, packed, mode, what):
    st, msg = _status("rsp_mask_paste", P, P, 3, HM, WM, *geo, *out_hw, *slot, packed, 0.5, mode)
    assert st == 1 and what in msg, msg


@pytest.mark.parametrize("geo, out_hw, slot, packed, what", [
    (GEO1, (48, 64), (48, 64), 1, "x4"),           # bits after one resize that is not x4
    (GEO1, (64, 64), (64, 80), 1, "x4"),           # x4 bits into larger slots
    (GEO1, (64, 64), (80, 64), 0, "(Hr, Wr)"),     # bytes whose slot is not the mask
    (GEO2, (150, 200), (150, 200), 1, "Wr % 16"),  # two resizes into bits with an unaligned slot width
])
def test_query_postprocess_rejects_unsupported_combinations(geo, out_hw, slot, packed, what):
    st, msg = _status("rsp_query_postprocess", P, P, P, 3, HM, WM, *geo, *out_hw, *slot, packed, P, P, P, P)
    assert st == 1 and what in msg, msg


def test_sam_mask_stats_crop_rule_needs_iou():
    """The crop-edge rule is part of the keep flag, which exists only with iou."""
    H, W = 150, 200
    crop = (100, 50, 100 + W, 50 + H, 1000, 1000)    # crop box and scene: valid
    st, msg = _status("rsp_sam_mask_stats", P, 3, HM, WM, *GEO2, H, W, 0.0, 1.0, -1.0, None, 0.88, 0.95, *crop, P, P, P,
                      P, P)
    assert st == 1 and "iou" in msg, msg
