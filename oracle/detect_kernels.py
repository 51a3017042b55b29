"""Float64 restatements of the anchor head's and the necks' standalone kernels (include/rsp_b200.h).  TEST
INFRASTRUCTURE ONLY.

  * ``rpn_decode``: rsp_rpn_decode with and without img_shapes, sigmoid scores and delta2bbox boxes of the top-k
    anchors, with the ``w > min_size and h > min_size`` filter (restate_anchor.delta2bbox, grid_anchors);
  * ``bbox_cls_decode``: rsp_bbox_cls_decode with and without img_shapes, a (C + 1)-way softmax with the background
    last, per-class delta2bbox, ``score > thr`` and the padding RoIs masked;
  * ``roi_align``: rsp_roi_align_nhwc, torchvision's roi_align (aligned=True, sampling_ratio=0) in float64 on the level
    restate_anchor.map_roi_levels picks in fp32 (mmdet computes it in fp32); with a PE table the reference is
    roi_align(feat + pe), since RoIAlign is linear;
  * ``sin_fold``: rsp_sin_fold, sin(x[..., ::2]) + x[..., 1::2].

Tolerances follow oracle/decoder_kernels.py: U8 = 2^-8 for a bf16 result, U24 = 2^-24 per fp32 rounding.  The box
arithmetic of the kernels rounds every operation (no FMA contraction) except expf, so its bound is a few roundings of
the magnitudes involved."""
from __future__ import annotations

import torch

from . import restate_anchor as ra
from .decoder_kernels import D, U8, U24


# ---------------------------------------------------------------------------------------------------- box decoding
def delta2bbox_tol(rois: torch.Tensor, deltas: torch.Tensor, stds, wh_ratio_clip: float = 16 / 1000) -> torch.Tensor:
    """Bound on the fp32 delta2bbox of rsp_b200 (detect.cu delta2bbox_one) against float64, [n, 4] for rois [n, 4] and
    deltas [n, 4]: each of px, pw, dx, pw dx, gx rounds once (U24 of its magnitude), gw = pw expf(dw) carries expf's 2
    ulp, the clamped dw's rounding and two more roundings, and the corner adds one more.  Clipping to the image is
    1-Lipschitz, so the unclipped magnitudes bound the clipped result."""
    r, d = rois.to(D), deltas.to(D) * torch.tensor(stds, dtype=D, device=rois.device)
    mr = abs(torch.log(torch.tensor(wh_ratio_clip, dtype=D)).item())
    pxy = (r[:, :2] + r[:, 2:]) * 0.5
    pwh = r[:, 2:] - r[:, :2]
    dwh = d[:, 2:].clamp(-mr, mr)
    gxy = pxy + pwh * d[:, :2]
    gwh = pwh * dwh.exp()
    corner = gxy.abs() + 0.5 * gwh.abs()
    t = 4 * U24 * (pxy.abs() + (pwh * d[:, :2]).abs() + gxy.abs() + corner) + (6 + dwh.abs()) * U24 * gwh.abs()
    return torch.cat([t, t], dim=1) + 1e-30


def rpn_anchors(H: int, W: int, stride: int, base: torch.Tensor) -> torch.Tensor:
    """restate_anchor.grid_anchors in fp32 (base + shift rounds as the kernel's does), as float64 [H W A, 4]."""
    return ra.grid_anchors((H, W), stride, base.float().cpu()).to(D)


def rpn_decode(head_out: torch.Tensor, topk_idx: torch.Tensor, H: int, W: int, A: int, stride: int,
               base: torch.Tensor, img_shapes: torch.Tensor, min_size: float, stds=(1.0, 1.0, 1.0, 1.0),
               wh_ratio_clip: float = 16 / 1000):
    """rsp_rpn_decode: head_out fp32 [B H W, >= 5A] (columns [0, A) logits, [A, 5A) deltas a * 4 + k), topk_idx
    int64 [B, K] (anchor index (y W + x) A + a), img_shapes [B, 2] (h, w) -> (boxes [B, K, 4], scores [B, K],
    tol [B, K, 4], wh [B, K, 2]) in float64; filtered scores are -1.  wh: the float64 box widths and heights."""
    B, K = topk_idx.shape
    anchors = rpn_anchors(H, W, stride, base)
    boxes, scores, tols = [], [], []
    for b in range(B):
        idx = topk_idx[b].cpu().long()
        rows = head_out[b * H * W:(b + 1) * H * W].cpu().to(D)[idx // A]                   # [K, ld]
        a = idx % A
        logit = rows.gather(1, a.view(-1, 1)).view(-1)
        d = torch.stack([rows.gather(1, (A + 4 * a + k).view(-1, 1)).view(-1) for k in range(4)], dim=1)
        r = anchors[idx]
        shape = img_shapes[b].cpu().to(D).tolist()
        bx = ra.delta2bbox(r, d, stds, shape, wh_ratio_clip)
        boxes.append(bx)
        scores.append(torch.sigmoid(logit))
        tols.append(delta2bbox_tol(r, d, stds))
    boxes, scores, tols = torch.stack(boxes), torch.stack(scores), torch.stack(tols)
    wh = boxes[..., 2:] - boxes[..., :2]
    keep = (wh[..., 0] > min_size) & (wh[..., 1] > min_size)
    return boxes, torch.where(keep, scores, torch.full_like(scores, -1.0)), tols, wh


def bbox_cls_decode(cls: torch.Tensor, reg: torch.Tensor, rois: torch.Tensor, roi_valid, C: int,
                    img_shapes: torch.Tensor, thr: float, stds=(0.1, 0.1, 0.2, 0.2)):
    """rsp_bbox_cls_decode: cls [n, >= C + 1] (background last), reg [n, >= 4C], rois [n, 5] (image, x1, y1, x2, y2),
    roi_valid uint8 [n] or None, img_shapes [images, 2] (h, w) indexed by rois[:, 0] -> (scores [n C] with -1 where
    score <= thr or the RoI is padding, raw softmax scores [n C], boxes [n C, 4], labels [n C], box tol [n C, 4],
    score tol [n C]), float64."""
    n = rois.shape[0]
    logits = cls[:, :C + 1].cpu().to(D)
    p = torch.softmax(logits, dim=-1)
    s = p[:, :C].reshape(-1)
    dev = (logits - logits.amax(-1, keepdim=True)).abs()           # expf(logit - max): |logit - max| U24 relative
    stol = ((dev[:, :C] + C + 8) * U24 * p[:, :C]).reshape(-1) + 1e-30
    rr = rois.cpu().to(D)
    d = reg[:, :4 * C].cpu().to(D).reshape(n * C, 4)
    r = rr[:, 1:].repeat_interleave(C, dim=0)
    img = rr[:, 0].long().repeat_interleave(C)
    boxes = torch.empty(n * C, 4, dtype=D)
    for b in img.unique().tolist():
        m = img == b
        boxes[m] = ra.delta2bbox(r[m], d[m], stds, img_shapes[b].cpu().to(D).tolist())
    valid = s > thr
    if roi_valid is not None:
        valid &= roi_valid.cpu().bool().repeat_interleave(C)
    labels = torch.arange(C).repeat(n)
    return torch.where(valid, s, torch.full_like(s, -1.0)), s, boxes, labels, delta2bbox_tol(r, d, stds), stol


# ---------------------------------------------------------------------------------------------------- RoIAlign
def roi_levels(rois: torch.Tensor, num_levels: int, finest_scale: float = 56.0) -> torch.Tensor:
    """restate_anchor.map_roi_levels on the fp32 RoIs (mmdet's arithmetic), int64 [n]."""
    return ra.map_roi_levels(rois.float().cpu(), num_levels, finest_scale)


def roi_align(feats: list, rois: torch.Tensor, P: int, strides, pes: list | None = None, aligned: bool = True,
              level_shift: int = 0) -> torch.Tensor:
    """rsp_roi_align_nhwc: feats bf16 NHWC levels, rois fp32 [n, 5], pes fp32 [H, W, C] per level or None ->
    float64 [n, P P C] in (ph, pw, c) order.  aligned / level_shift restate defects (the half-pixel offset dropped,
    the level one off)."""
    if ra.tvops is None:
        raise RuntimeError("torchvision is needed for the RoIAlign reference")
    L, n, C = len(feats), rois.shape[0], feats[0].shape[3]
    dev = feats[0].device
    lv = (roi_levels(rois, L) + level_shift) % L
    out = torch.zeros(n, C, P, P, dtype=D, device=dev)
    r64 = rois.to(D).to(dev)
    for i in range(L):
        idx = (lv == i).nonzero(as_tuple=False).view(-1).to(dev)
        if idx.numel() == 0:
            continue
        f = feats[i].to(D).permute(0, 3, 1, 2)
        if pes is not None:
            f = f + pes[i].to(D).permute(2, 0, 1).unsqueeze(0)
        out[idx] = ra.tvops.roi_align(f, r64[idx], P, spatial_scale=1.0 / strides[i], sampling_ratio=0,
                                      aligned=aligned)
    return out.permute(0, 2, 3, 1).reshape(n, P * P * C)


def roi_sample_positions(rois: torch.Tensor, scale: torch.Tensor, P: int, dtype=D):
    """The sample coordinates of every RoI with the kernel's operation order in ``dtype``: (ys [n, P, gh_max],
    xs [n, P, gw_max]) padded with NaN, and (gh, gw) [n].  scale [n]: the RoI's level scale (1 / stride)."""
    r = rois.cpu().to(dtype)
    ss = scale.cpu().to(dtype)
    x1, y1 = r[:, 1] * ss - 0.5, r[:, 2] * ss - 0.5
    rw, rh = (r[:, 3] * ss - 0.5) - x1, (r[:, 4] * ss - 0.5) - y1
    bw, bh = rw / P, rh / P
    gh, gw = torch.ceil(rh / P).clamp(min=0).long(), torch.ceil(rw / P).clamp(min=0).long()
    gmax = max(1, int(gh.max()), int(gw.max()))
    p = torch.arange(P, dtype=dtype).view(1, P, 1)
    i = torch.arange(gmax, dtype=dtype).view(1, 1, gmax) + 0.5
    ys = y1.view(-1, 1, 1) + p * bh.view(-1, 1, 1) + i * bh.view(-1, 1, 1) / gh.clamp(min=1).to(dtype).view(-1, 1, 1)
    xs = x1.view(-1, 1, 1) + p * bw.view(-1, 1, 1) + i * bw.view(-1, 1, 1) / gw.clamp(min=1).to(dtype).view(-1, 1, 1)
    ys = torch.where(i < gh.view(-1, 1, 1), ys, torch.full_like(ys, float("nan")))
    xs = torch.where(i < gw.view(-1, 1, 1), xs, torch.full_like(xs, float("nan")))
    return ys, xs, gh, gw


def roi_edge_gap(rois: torch.Tensor, sizes, strides, P: int) -> torch.Tensor:
    """Per RoI, the smallest float64 distance of a sample to RoIAlign's discontinuities y = -1, y = H, x = -1, x = W
    (a sample past them reads 0, a sample on them the clamped border pixel), samples exactly on them excluded: [n]."""
    L = len(sizes)
    lv = roi_levels(rois, L)
    scale = torch.tensor([1.0 / strides[l] for l in lv.tolist()], dtype=D)
    hs = torch.tensor([float(sizes[l][0]) for l in lv.tolist()], dtype=D).view(-1, 1, 1)
    ws = torch.tensor([float(sizes[l][1]) for l in lv.tolist()], dtype=D).view(-1, 1, 1)
    ys, xs, _, _ = roi_sample_positions(rois, scale, P)
    gaps = [(ys + 1).abs(), (ys - hs).abs(), (xs + 1).abs(), (xs - ws).abs()]
    gaps = [torch.where((g == 0) | g.isnan(), torch.full_like(g, float("inf")), g).flatten(1).amin(1) for g in gaps]
    return torch.stack(gaps, dim=1).amin(1)


def roi_align_tol(feats: list, rois: torch.Tensor, P: int, strides, ref: torch.Tensor,
                  pes: list | None = None) -> torch.Tensor:
    """Bound on |kernel - roi_align|, [n, P P C].  With F = max |feat| (+ max |pe|) of the RoI's level:
      * sample positions: y1 + ph bh + (iy + 1/2) bh / gh in fp32 is within 24 U24 m of float64, m = the RoI's largest
        coordinate on the level grid + 1; RoIAlign's bilinear sample is continuous away from -1 and H / W (kept off
        those by the inputs, or exactly on them in fp32 too), with slope <= 2 F per axis;
      * the fp32 sum over gh gw samples of 4 corners (and the PE's), then / count: (gh gw + 8) U24 F;
      * the bf16 output: U8 |ref|."""
    L, n, C = len(feats), rois.shape[0], feats[0].shape[3]
    lv = roi_levels(rois, L)
    fmax = torch.tensor([feats[l].abs().max().item() + (0.0 if pes is None else pes[l].abs().max().item())
                         for l in range(L)], dtype=D)[lv]
    scale = torch.tensor([1.0 / strides[l] for l in lv.tolist()], dtype=D)
    r = rois.cpu().to(D)
    m = r[:, 1:].abs().amax(1) * scale + 1
    _, _, gh, gw = roi_sample_positions(rois, scale, P)
    cnt = (gh * gw).clamp(min=1).to(D)
    per = (2 * 2 * 24 * U24 * m + (cnt + 8) * U24) * fmax + 1e-30
    per = per.to(ref.device).view(n, 1).expand(n, P * P * C)
    return per * (1 + U8) + U8 * ref.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------- sin fold
def ulp32(v: torch.Tensor) -> torch.Tensor:
    """fp32 ulp of |v| (float64 v), 2^-149 at least."""
    e = torch.floor(torch.log2(v.abs().clamp(min=2.0 ** -126)))
    return torch.pow(2.0, e - 23).to(D).clamp(min=2.0 ** -149)


def sin_fold(x: torch.Tensor):
    """rsp_sin_fold: fp32 [..., 2k] -> (float64 [..., k] sin(x[..., ::2]) + x[..., 1::2], tol): sinf is within 2 ulp
    of sin over the whole fp32 range (CUDA's documented bound), then the add rounds once."""
    s = torch.sin(x[..., ::2].to(D))
    ref = s + x[..., 1::2].to(D)
    return ref, 2 * ulp32(s) + ulp32(ref)


# ---------------------------------------------------------------------------------------------------- input builders
def rpn_inputs(B: int, H: int, W: int, A: int, K: int, ld: int, seed: int):
    """head_out fp32 [B H W, ld] (ld > 5A: the columns past 5A are never read), topk_idx int64 [B, K] with the first
    and last anchor in every image.  Logits N(0, 4); dx, dy N(0, 1.5); a third of dw, dh beyond +-log(1000 / 16) of
    either sign (the wh_ratio_clip clamp), the rest N(0, 1), so boxes cross the image border."""
    g = torch.Generator().manual_seed(seed)
    head = torch.randn(B * H * W, ld, generator=g)
    head[:, :A] *= 4
    d = head[:, A:5 * A].reshape(-1, A, 4)
    d[..., :2] *= 1.5
    big = torch.rand(B * H * W, A, 2, generator=g) < 1 / 3
    sgn = torch.where(torch.rand(B * H * W, A, 2, generator=g) < 0.5, -1.0, 1.0)
    d[..., 2:] = torch.where(big, sgn * (4.2 + 3 * torch.rand(B * H * W, A, 2, generator=g)), d[..., 2:])
    head[:, A:5 * A] = d.reshape(-1, 4 * A)
    n = H * W * A
    idx = torch.stack([torch.cat([torch.tensor([0, n - 1]), torch.randperm(n - 2, generator=g)[:K - 2] + 1])
                       for _ in range(B)])
    return head.contiguous(), idx.contiguous()


def bbox_inputs(n: int, C: int, ld_cls: int, images: int, img_hw: tuple, seed: int):
    """cls fp32 [n, ld_cls] (logits up to +-60), reg fp32 [n, 4C + 4] (dw, dh beyond the clamp for some), rois fp32
    [n, 5] spread over ``images`` images and across the image border, roi_valid uint8 [n] with zeros."""
    g = torch.Generator().manual_seed(seed)
    cls = 6 * torch.randn(n, ld_cls, generator=g)
    cls[::7] *= 10                                           # some rows with logits up to about +-60
    cls = cls.clamp(-60, 60)
    reg = torch.randn(n, 4 * C + 4, generator=g) * 2
    reg[::5, 2::4] = 30 * torch.sign(reg[::5, 2::4])         # dw / dh * 0.2 beyond +-4.14
    H, W = img_hw
    cx, cy = torch.rand(n, generator=g) * (W + 100) - 50, torch.rand(n, generator=g) * (H + 100) - 50
    bw, bh = torch.exp(torch.rand(n, generator=g) * 6), torch.exp(torch.rand(n, generator=g) * 6)
    img = torch.randint(0, images, (n,), generator=g).float()
    rois = torch.stack([img, cx - bw, cy - bh, cx + bw, cy + bh], dim=1)
    valid = (torch.rand(n, generator=g) > 0.2).to(torch.uint8)
    return cls.contiguous(), reg.contiguous(), rois.contiguous(), valid


def roi_inputs(B: int, C: int, img: int, strides, seed: int, pe: bool):
    """Four NHWC levels bf16 [B, img / s, img / s, C] with per-level offsets, PE tables fp32 [H, W, C] (or None) and
    the RoIs (fp32 [n, 5], both images):
      sub-pixel RoIs; the whole image; partly and fully outside the map; zero width, zero height and a point; sqrt(area)
      exactly 112, 224 and 448 (the level boundaries of finest_scale 56) and a non-square 64 x 196 at 112; samples
      exactly on y = -1, y = H, x = -1 and x = W of level 0 (exact in fp32: bins of one pixel); random RoIs whose
      samples keep > 1e-3 from those edges."""
    g = torch.Generator().manual_seed(seed)
    sizes = [(img // s, img // s) for s in strides]
    feats = [(torch.randn(B, h, w, C, generator=g) + l).to(torch.bfloat16) for l, (h, w) in enumerate(sizes)]
    pes = [torch.randn(h, w, C, generator=g) * 0.5 for h, w in sizes] if pe else None
    fixed = [
        (100.3, 200.7, 100.9, 201.2), (512.25, 3.5, 513.0, 4.0),            # sub-pixel
        (0.0, 0.0, img, img), (0.0, 0.0, img - 0.5, 700.0),                  # whole image
        (-50.0, 900.0, 60.0, 1100.0), (980.0, -30.0, 1100.0, 40.0),          # partly outside
        (-300.0, -300.0, -200.0, -250.0), (1100.0, 1100.0, 1300.0, 1200.0),  # fully outside
        (500.0, 300.0, 500.0, 400.0), (10.0, 20.0, 80.0, 20.0), (5.0, 5.0, 5.0, 5.0),   # zero width / height
        (200.0, 300.0, 312.0, 412.0), (100.0, 100.0, 324.0, 324.0), (300.0, 200.0, 748.0, 648.0),   # 112, 224, 448
        (0.5, 10.0, 64.5, 206.0),                                           # 64 x 196: sqrt(area) = 112
        (400.0, 1000.0, 428.0, 1028.0), (-4.0, -4.0, 24.0, 24.0),           # samples on y = H / x, y = -1 (level 0)
        (1000.0, 400.0, 1028.0, 428.0),                                      # samples on x = W
    ]
    rois = [(b, *r) for r in fixed for b in range(B)]
    out = torch.tensor(rois, dtype=torch.float32)
    want = 64
    rnd = []
    while len(rnd) < want:
        c = torch.rand(2, generator=g) * (img + 200) - 100
        wh = torch.exp(torch.rand(2, generator=g) * 6.5)
        r = torch.tensor([[float(len(rnd) % B), c[0] - wh[0], c[1] - wh[1], c[0] + wh[0], c[1] + wh[1]]])
        if roi_edge_gap(r, sizes, strides, 7).item() > 1e-3 and roi_edge_gap(r, sizes, strides, 14).item() > 1e-3:
            rnd.append(r)
    return feats, pes, torch.cat([out] + rnd).contiguous(), sizes
