"""The anchor head's and the necks' standalone kernels one by one against oracle/detect_kernels.py.

Box coordinates and scores are held to bounds derived from the kernels' rounding points (a few fp32 roundings of the
magnitudes involved: the box arithmetic rounds every operation but expf), RoIAlign to its float64 bound, and the
integer-valued results (labels, the score filters, max pooling, the bf16 table add) must match exactly.  Each case
prints max|err| and max|err|/tol."""
import pytest
import torch
import torch.nn.functional as F

from oracle import detect_kernels as dtk
from oracle import restate_anchor as ra

pytestmark = pytest.mark.gpu

STRIDES = [4, 8, 16, 32]


def _check(out, ref, tol, what):
    err = (out.to(torch.float64).cpu() - ref.cpu()).abs()
    ratio = (err / tol.cpu()).max().item()
    print(f"{what}: max|err| {err.max().item():.3e}  max|err|/tol {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: max |err| / tol = {ratio:.3f}, max |err| = {err.max().item():.3e}"


@pytest.mark.parametrize("per_image", [False, True])
def test_rpn_decode(per_image):
    """A = 3 on a 24 x 40 map, B = 2, head_out with ld = 19 > 5A; the first and last anchor among the top-k; |dw|,
    |dh| beyond log(1000 / 16) of both signs; boxes across the image border; a scalar image shape or one per image.
    The output sits at out_off = 7 of a wider list prefilled with a sentinel that must survive outside [7, 7 + K).

    The min-size filter must agree exactly, except where a float64 width or height lies within 1e-4 (or the two
    coordinates' tolerance, if larger) of min_size: there the kernel's fp32 width may fall on either side."""
    from rsprompter_b200 import _lib
    B, H, W, A, K, off, n_tot, min_size = 2, 24, 40, 3, 600, 7, 640, 2.0
    head, idx = dtk.rpn_inputs(B, H, W, A, K, ld=5 * A + 4, seed=5 + per_image)
    base = ra.base_anchors(16, (8,), (0.5, 1.0, 2.0))
    shapes = torch.tensor([[384.0, 640.0], [300.0, 500.0]]) if per_image else torch.tensor([[384.0, 640.0]] * B)
    boxes = torch.full((B, n_tot, 4), 12345.0, device="cuda")
    scores = torch.full((B, n_tot), 12345.0, device="cuda")
    _lib.rpn_decode(head.cuda(), idx.cuda(), B, H, W, A, 16, base.cuda(), (384, 640), min_size, boxes, scores, off,
                    img_shapes=shapes.cuda() if per_image else None)
    torch.cuda.synchronize()
    boxes, scores = boxes.cpu(), scores.cpu()
    outside = torch.ones(n_tot, dtype=torch.bool)
    outside[off:off + K] = False
    assert (boxes[:, outside] == 12345.0).all() and (scores[:, outside] == 12345.0).all()
    rb, rs, tol, wh = dtk.rpn_decode(head, idx, H, W, A, 16, base, shapes, min_size)
    what = f"rpn_decode {'img_shapes' if per_image else 'img_hw'}"
    _check(boxes[:, off:off + K], rb, tol, what + " boxes")
    margin = torch.maximum(tol[..., :2] + tol[..., 2:], torch.full_like(wh, 1e-4))
    edge = ((wh - min_size).abs() <= margin).any(-1)
    got = scores[:, off:off + K]
    kf, rf = got == -1, rs == -1
    print(f"{what}: {int(rf.sum())} of {B * K} filtered, {int(edge.sum())} within the margin of min_size")
    assert rf.any() and (~rf).any()
    assert torch.equal(kf[~edge], rf[~edge])
    both = ~kf & ~rf
    _check(got[both], rs[both], 4 * dtk.U24 * rs[both] + 1e-30, what + " scores")


@pytest.mark.parametrize("C", [10, 1])
@pytest.mark.parametrize("per_image", [False, True])
def test_bbox_cls_decode(C, per_image):
    """C + 1-way softmax with ld_cls = C + 3, logits up to +-60, padding RoIs (roi_valid 0), per-image shapes through
    rois[:, 0].  Labels are exact; the score filter is exact away from thr +- 1e-6."""
    from rsprompter_b200 import _lib
    n, thr = 300, 0.05
    cls, reg, rois, valid = dtk.bbox_inputs(n, C, C + 3, 2, (600, 800), seed=10 * C + per_image)
    shapes = torch.tensor([[600.0, 800.0], [480.0, 700.0]]) if per_image else torch.tensor([[600.0, 800.0]] * 2)
    s, bx, lab = _lib.bbox_cls_decode(cls.cuda(), reg.cuda(), rois.cuda(), valid.cuda(), C, (600, 800), thr,
                                      img_shapes=shapes.cuda() if per_image else None)
    torch.cuda.synchronize()
    s, bx, lab = s.cpu(), bx.cpu(), lab.cpu()
    ref_s, raw, ref_b, ref_l, btol, stol = dtk.bbox_cls_decode(cls, reg, rois, valid, C, shapes, thr)
    what = f"bbox_cls_decode C={C} {'img_shapes' if per_image else 'img_hw'}"
    assert torch.equal(lab, ref_l)
    _check(bx, ref_b, btol, what + " boxes")
    edge = (raw - thr).abs() <= 1e-6
    kf, rf = s == -1, ref_s == -1
    assert rf.any() and (~rf).any() and (valid == 0).any()
    assert torch.equal(kf[~edge], rf[~edge])
    both = ~kf & ~rf
    _check(s[both], raw[both], stol[both], what + " scores")


@pytest.mark.skipif(ra.tvops is None, reason="torchvision is not installed")
@pytest.mark.parametrize("P", [7, 14])
@pytest.mark.parametrize("pe", [False, True])
def test_roi_align_nhwc(P, pe):
    """Four levels (strides 4 .. 32 of a 1024 image), C = 256, B = 2 with RoIs of both images: sub-pixel and
    whole-image RoIs, RoIs partly and fully outside the map, zero width / height (exactly 0, count 1), sqrt(area)
    exactly 112, 224 and 448 (level boundaries), samples exactly on y = -1 / H and x = -1 / W, random RoIs; with and
    without the per-level PE tables (reference: RoIAlign of feat + pe)."""
    from rsprompter_b200 import _lib
    feats, pes, rois, _ = dtk.roi_inputs(2, 256, 1024, STRIDES, seed=P + pe, pe=pe)
    feats = [f.cuda() for f in feats]
    pes = None if pes is None else [p.cuda() for p in pes]
    out = _lib.roi_align_nhwc(feats, rois.cuda(), P, STRIDES, pes)
    torch.cuda.synchronize()
    ref = dtk.roi_align(feats, rois, P, STRIDES, pes)
    zero = (rois[:, 1] == rois[:, 3]) | (rois[:, 2] == rois[:, 4])
    assert (out[zero.cuda()] == 0).all()
    _check(out, ref, dtk.roi_align_tol(feats, rois, P, STRIDES, ref, pes), f"roi_align P={P} pe={pe}")


@pytest.mark.parametrize("mode", [0, 1])
def test_pool2_nhwc(mode):
    """Mode 0: MaxPool2d(2, 2); mode 1: max_pool2d(k=1, s=2); odd H and W, bitwise against F.max_pool2d."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(mode)
    x = (torch.randn(2, 33, 47, 64, generator=g) * 3).to(torch.bfloat16).cuda()
    out = _lib.pool2_nhwc(x, mode)
    torch.cuda.synchronize()
    k = 2 if mode == 0 else 1
    exp = F.max_pool2d(x.permute(0, 3, 1, 2), k, 2).permute(0, 2, 3, 1)
    assert out.shape == exp.shape and torch.equal(out, exp)


def test_sin_fold():
    """sin(x[..., ::2]) + x[..., 1::2] for |x| up to 1e4 (the sine PE range), within sinf's 2 ulp and one rounding."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(0)
    x = ((torch.rand(5000, 2, generator=g) * 2 - 1) * torch.logspace(-3, 4, 5000).view(-1, 1)).reshape(50, 5, 40)
    x = x.float().cuda()
    out = _lib.sin_fold(x)
    torch.cuda.synchronize()
    ref, tol = dtk.sin_fold(x)
    _check(out, ref, tol, "sin_fold")


def test_add_table_bf16():
    """bf16 x [3, 5, 72] + fp32 table [5, 72] (period 360 = 8 x 45) -> bf16, bitwise against bf16(x.float() + table)."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(3, 5, 72, generator=g) * 4).to(torch.bfloat16).cuda()
    table = torch.randn(5, 72, generator=g).cuda()
    out = _lib.add_table_bf16(x, table)
    torch.cuda.synchronize()
    assert torch.equal(out, (x.float() + table).to(torch.bfloat16))
