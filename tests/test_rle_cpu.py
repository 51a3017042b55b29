"""Argument checks of the COCO RLE entry points that run before any launch, so they hold without a GPU: a mask must
have 1 .. 2^31 - 1 pixels."""
import ctypes

import pytest

from rsprompter_b200 import _lib


@pytest.mark.parametrize("h, w", [(46341, 46341), (1, 2 ** 31), (0, 5), (5, 0), (-1, 4)])
def test_mask_rle_rejects_bad_mask_sizes(h, w):
    desc = (ctypes.c_int64 * 6)(0, 4, 4, 16, h, w)          # mask 0 is valid, mask 1 is not
    fake = ctypes.c_void_p(16)                               # never dereferenced: the check precedes every launch
    status = _lib._lib.rsp_mask_rle_lengths(fake, 0, fake, ctypes.cast(desc, ctypes.c_void_p), 2, fake, None)
    assert status == 1
    assert b"mask 1" in _lib._lib.rsp_last_error()

