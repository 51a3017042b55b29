"""The float64 references of the anchor head's and the necks' kernels (oracle/detect_kernels.py), checked without a
GPU:
  * pinned to the fp32 restatements they stand in for (restate_anchor's grid_anchors / delta2bbox / sigmoid / softmax
    and roi_extract, the sin fold of mask_head_prompts); the fp32 restatement also lands inside each tolerance, so
    the bounds are not tighter than one more fp32 evaluation;
  * bug distance: on the inputs of tests/test_detect_kernels_gpu.py, delta2bbox without its wh_ratio_clip clamp and
    RoIAlign with aligned=False or its level one off land more than 10x the tolerance away, so the GPU test would
    fail on them;
  * the RoIs keep their samples off RoIAlign's discontinuities, or exactly on them in fp32 as in float64."""
import pytest
import torch

from oracle import decoder_kernels as dk
from oracle import detect_kernels as dtk
from oracle import restate_anchor as ra

FAR = 10.0
STRIDES = (4, 8, 16, 32)
needs_tv = pytest.mark.skipif(ra.tvops is None, reason="torchvision is not installed")


def _far(bug, ref, tol, what):
    r = dk.max_ratio((bug - ref).abs(), tol)
    assert r > FAR, f"{what}: the defect is only {r:.1f} x the tolerance away"


def _rpn_case(B=2, H=24, W=40, A=3, K=400):
    head, idx = dtk.rpn_inputs(B, H, W, A, K, ld=5 * A + 4, seed=1)
    base = ra.base_anchors(16, (8,), (0.5, 1.0, 2.0))
    shapes = torch.tensor([[384.0, 640.0], [300.0, 500.0]])
    return head, idx, base, shapes, (B, H, W, A)


def test_rpn_decode_matches_fp32_restatement():
    """restate_anchor's fp32 grid_anchors + delta2bbox + sigmoid (rpn_predict_single's arithmetic) on the same top-k
    anchors land inside the float64 reference's tolerance."""
    head, idx, base, shapes, (B, H, W, A) = _rpn_case()
    boxes, scores, tol, _ = dtk.rpn_decode(head, idx, H, W, A, 16, base, shapes, 0.0)
    pri = ra.grid_anchors((H, W), 16, base)
    for b in range(B):
        rows = head[b * H * W:(b + 1) * H * W]
        cls = rows[:, :A].reshape(-1)
        reg = rows[:, A:5 * A].reshape(-1, 4)
        bx = ra.delta2bbox(pri[idx[b]], reg[idx[b]], (1.0, 1.0, 1.0, 1.0), tuple(shapes[b].tolist()))
        assert dk.max_ratio((bx.double() - boxes[b]).abs(), tol[b]) <= 1.0
        assert dk.max_ratio((cls[idx[b]].sigmoid().double() - scores[b]).abs(), 4 * dk.U24 * scores[b] + 1e-30) <= 1.0


def test_rpn_decode_without_clamp_is_far():
    head, idx, base, shapes, (B, H, W, A) = _rpn_case()
    boxes, _, tol, _ = dtk.rpn_decode(head, idx, H, W, A, 16, base, shapes, 0.0)
    bug, _, _, _ = dtk.rpn_decode(head, idx, H, W, A, 16, base, shapes, 0.0, wh_ratio_clip=1e-300)
    _far(bug, boxes, tol, "delta2bbox without the wh_ratio_clip clamp")


@pytest.mark.parametrize("C", [10, 1])
def test_bbox_cls_decode_matches_fp32_restatement(C):
    """bbox_predict_single's fp32 softmax and per-class delta2bbox land inside the tolerance; labels are the class of
    each column; scores <= thr and padding RoIs are -1."""
    cls, reg, rois, valid = dtk.bbox_inputs(300, C, C + 3, 2, (600, 800), seed=C)
    shapes = torch.tensor([[600.0, 800.0], [480.0, 700.0]])
    scores, raw, boxes, labels, btol, stol = dtk.bbox_cls_decode(cls, reg, rois, valid, C, shapes, 0.05)
    p = torch.softmax(cls[:, :C + 1], dim=-1)[:, :C].reshape(-1)
    assert dk.max_ratio((p.double() - raw).abs(), stol) <= 1.0
    for b in (0, 1):
        m = (rois[:, 0] == b).repeat_interleave(C)
        r = rois[:, 1:].repeat_interleave(C, dim=0)[m]
        bx = ra.delta2bbox(r, reg[:, :4 * C].reshape(-1, 4)[m], (0.1, 0.1, 0.2, 0.2), tuple(shapes[b].tolist()))
        assert dk.max_ratio((bx.double() - boxes[m]).abs(), btol[m]) <= 1.0
    assert torch.equal(labels, torch.arange(C).repeat(300))
    assert ((scores == -1) == ((raw <= 0.05) | (valid == 0).repeat_interleave(C))).all()
    _far(torch.cat([ra.delta2bbox(rois[i:i + 1, 1:].double(), reg[i:i + 1, :4 * C].double(), (0.1, 0.1, 0.2, 0.2),
                                  tuple(shapes[int(rois[i, 0])].tolist()), 1e-300).view(C, 4)
                    for i in range(300)]), boxes, btol, "delta2bbox without the wh_ratio_clip clamp")


@needs_tv
def test_roi_align_matches_roi_extract():
    """roi_align is restate_anchor.roi_extract (SingleRoIExtractor on torchvision's RoIAlign) in float64, and a
    zero-width RoI gives 0."""
    feats, pes, rois, _ = dtk.roi_inputs(2, 8, 1024, STRIDES, seed=1, pe=True)
    ref = dtk.roi_align(feats, rois, 7, STRIDES, pes)
    nchw = [(f.float() + p.unsqueeze(0)).permute(0, 3, 1, 2) for f, p in zip(feats, pes)]
    exp = ra.roi_extract(nchw, rois, 7, STRIDES).permute(0, 2, 3, 1).reshape(rois.shape[0], -1)
    assert (ref - exp.double()).abs().max().item() < 2e-5 * exp.abs().max().item()
    zero = (rois[:, 1] == rois[:, 3]) | (rois[:, 2] == rois[:, 4])
    assert zero.sum() >= 6 and (ref[zero] == 0).all()


@needs_tv
@pytest.mark.parametrize("P", [7, 14])
def test_roi_align_defects_are_far(P):
    feats, pes, rois, _ = dtk.roi_inputs(2, 8, 1024, STRIDES, seed=P, pe=P == 7)
    ref = dtk.roi_align(feats, rois, P, STRIDES, pes)
    tol = dtk.roi_align_tol(feats, rois, P, STRIDES, ref, pes)
    _far(dtk.roi_align(feats, rois, P, STRIDES, pes, aligned=False), ref, tol, "aligned=False")
    _far(dtk.roi_align(feats, rois, P, STRIDES, pes, level_shift=1), ref, tol, "level one off")


@pytest.mark.parametrize("P", [7, 14])
def test_roi_samples_avoid_the_edges(P):
    """Every sample of the test RoIs lies more than 1e-3 from y = -1, y = H, x = -1 and x = W of its level, or exactly
    on one of them in fp32 (the kernel's operation order) as in float64; some lie exactly on each."""
    _, _, rois, sizes = dtk.roi_inputs(2, 8, 1024, STRIDES, seed=P, pe=False)
    assert (dtk.roi_edge_gap(rois, sizes, STRIDES, P) > 1e-3).all()
    lv = dtk.roi_levels(rois, 4)
    scale = torch.tensor([1.0 / STRIDES[l] for l in lv.tolist()], dtype=torch.float64)
    ys64, xs64, _, _ = dtk.roi_sample_positions(rois, scale, P)
    ys32, xs32, _, _ = dtk.roi_sample_positions(rois, scale.float(), P, dtype=torch.float32)
    H = torch.tensor([float(sizes[l][0]) for l in lv.tolist()], dtype=torch.float64).view(-1, 1, 1)
    for s64, s32 in ((ys64, ys32), (xs64, xs32)):
        on = (s64 == -1) | (s64 == H)
        assert torch.equal(s32.double()[on], s64[on])
    if P == 7:
        assert ((ys64 == -1).any() and (ys64 == H).any() and (xs64 == -1).any() and (xs64 == H).any())


def test_sin_fold_matches_restate():
    """mask_head_prompts' fp32 fold lands within the tolerance of the float64 reference up to |x| = 1e4."""
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(4000, 2, generator=g) * 2 - 1) * torch.logspace(-3, 4, 4000).view(-1, 1)
    x = x.reshape(40, 200).float()
    ref, tol = dtk.sin_fold(x)
    assert dk.max_ratio((torch.sin(x[..., ::2]) + x[..., 1::2]).double().sub(ref).abs(), tol) <= 1.0
