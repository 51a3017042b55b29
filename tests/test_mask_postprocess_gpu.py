"""Cross-layout identities of the mask post-processing entry points: the bit-packed record layouts hold exactly the
bits of the byte layouts, and mode 0's in-kernel sigmoid equals rsp_sigmoid_f32 followed by mode 2.  The entry points
are called through the C ABI, so the identities pin the kernels whatever the Python wrappers look like."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BATCH, CROP = (256, 256), (200, 240)


def _c(name, *args):
    from rsprompter_b200 import _lib
    _lib._check(getattr(_lib._lib, "rsp_" + name)(*[_lib._ptr(a) if isinstance(a, torch.Tensor) else a for a in args],
                                                  _lib._stream()), "rsp_" + name)


def _logits(n, hm, wm, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, hm, wm, generator=g) * 3).cuda()


def _u8(*shape):
    return torch.empty(*shape, dtype=torch.uint8, device="cuda")


def _slot_bits(bytes_, Hr, Wr):
    """bytes [n, H, W] -> record slots [n, Hr, Wr/8] with the mask at the top-left and 0 elsewhere."""
    from rsprompter_b200 import _lib
    n, H, W = bytes_.shape
    full = torch.zeros(n, Hr, Wr, dtype=torch.uint8, device="cuda")
    full[:, :H, :W] = bytes_
    return _lib.pack_mask_bits(full)


@pytest.mark.parametrize("ori", [(150, 200), (151, 203), (97, 61)])
@pytest.mark.parametrize("mode", [1, 2])
def test_paste_two_resize_bits_equal_packed_bytes(ori, mode):
    """rsp_mask_paste through two resizes into bits in (H, round_up16(W)) slots and in larger slots equals its bytes,
    packed; at odd W the bits past column W are 0."""
    H, W = ori
    maps = _logits(5, 64, 64, H * W + mode)
    thr = 0.0 if mode == 1 else 0.5
    if mode == 2:
        maps = maps.sigmoid().contiguous()
    geo = (64, 64, *BATCH, *CROP, H, W)
    bytes_ = _u8(5, H, W)
    _c("mask_paste", maps, bytes_, 5, *geo, H, W, 0, thr, mode)
    assert 0 < bytes_.sum() < bytes_.numel()
    for Hr, Wr in [(H, (W + 15) // 16 * 16), (H + 9, (W + 15) // 16 * 16 + 32)]:
        bits = _u8(5, Hr, Wr // 8)
        _c("mask_paste", maps, bits, 5, *geo, Hr, Wr, 1, thr, mode)
        assert torch.equal(bits, _slot_bits(bytes_, Hr, Wr))


@pytest.mark.parametrize("ori", [(150, 200), (151, 203)])
def test_query_two_resize_bits_equal_packed_bytes(ori):
    """rsp_query_postprocess through two resizes: the bits are its packed bytes, and the scores and boxes are
    identical, also for slots with more rows than the mask."""
    H, W = ori
    logits = _logits(9, 64, 64, W)
    sel = torch.tensor([3, 0, 8, 3, 5, 5], dtype=torch.int32, device="cuda")
    cls = torch.rand(6, generator=torch.Generator().manual_seed(1)).cuda()
    n = sel.numel()
    geo = (64, 64, *BATCH, *CROP, H, W)
    bytes_ = _u8(n, H, W)
    part = torch.empty(n * ((H + 15) // 16) * 6, device="cuda")
    s0, b0 = torch.empty(n, device="cuda"), torch.empty(n, 4, device="cuda")
    _c("query_postprocess", logits, sel, cls, n, *geo, H, W, 0, bytes_, part, s0, b0)
    assert 0 < bytes_.sum() < bytes_.numel()
    for Hr, Wr in [(H, (W + 15) // 16 * 16), (H + 40, (W + 15) // 16 * 16 + 16)]:
        bits = _u8(n, Hr, Wr // 8)
        part = torch.empty(n * ((Hr + 15) // 16) * 6, device="cuda")
        s1, b1 = torch.empty(n, device="cuda"), torch.empty(n, 4, device="cuda")
        _c("query_postprocess", logits, sel, cls, n, *geo, Hr, Wr, 1, bits, part, s1, b1)
        assert torch.equal(bits, _slot_bits(bytes_, Hr, Wr))
        assert torch.equal(s0, s1) and torch.equal(b0, b1)


def test_paste_boxes_packed_equals_packed_bytes():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(3)
    probs = torch.rand(6, 28, 28, generator=g).cuda()
    boxes = torch.tensor([[10., 20., 200., 150.], [50., 50., 50., 90.], [-40., -30., 60., 70.],
                          [300., 10., 420., 300.], [500., 500., 600., 600.], [0., 0., 320., 320.]]).cuda()
    bytes_ = _lib.mask_paste_boxes(probs, boxes, (256, 320), 0.5)
    bits = _u8(6, 256, 40)
    _lib.mask_paste_boxes(probs, boxes, (256, 320), 0.5, bits=bits)
    assert 0 < bytes_.sum() < bytes_.numel()
    assert torch.equal(bits, _lib.pack_mask_bits(bytes_))


@pytest.mark.parametrize("shape,size", [((3, 5, 7), (24, 32)), ((1, 9, 13), (16, 48)), ((2, 15, 11), (64, 16))])
def test_paste_one_resize_mode0_equals_sigmoid_then_mode2(shape, size):
    """n * hm * wm not divisible by 4: rsp_mask_paste's mode 0 activates the taps in the kernel, with the arithmetic of
    rsp_sigmoid_f32 followed by mode 2."""
    from rsprompter_b200 import _lib
    n, hm, wm = shape
    logits = _logits(n, hm, wm, hm * wm)
    assert logits.numel() % 4
    got, ref = _u8(n, *size), _u8(n, *size)
    _c("mask_paste", logits, got, n, hm, wm, 0, 0, 0, 0, *size, *size, 0, 0.5, 0)
    pad = torch.zeros((logits.numel() + 3) // 4 * 4, device="cuda")
    pad[:logits.numel()] = logits.reshape(-1)
    act = _lib.sigmoid_f32(pad)
    _c("mask_paste", act, ref, n, hm, wm, 0, 0, 0, 0, *size, *size, 0, 0.5, 2)
    assert 0 < ref.sum() < ref.numel()
    assert torch.equal(got, ref)
