"""Generates tests/golden/reference_panoptic.pt by EXECUTING the reference's own panoptic post-processing:
MaskFormerFusionHead.panoptic_postprocess (mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py:41-106)
and RSMaskFormerFusionHead.predict (mmdet/rsprompter/models.py:663-715), pulled out of the reference tree with
make_golden.load_defs (nothing is copied into this repo).  INSTANCE_OFFSET and a PixelData stub are injected into their
namespace; `self` is a SimpleNamespace.
Run in the build container:   python tests/golden/make_golden_panoptic.py
The fixture pins oracle/restate_panoptic.py in tests/test_panoptic_cpu.py and the kernels in tests/test_panoptic_gpu.py.

Every case is one image of NQ queries on a 24 x 32 map.  Query 0 is an absorber: kept, logit -5 everywhere, so it wins
every pixel no designed region claims, and it is skipped (original_area 0), which leaves those pixels at num_classes.
Designed queries have logit -20 outside their regions.
"""
import os
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import load_defs  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_panoptic.pt")
H, W = 24, 32
C, THINGS = 5, 3          # labels 0-2 things, 3-4 stuff, 5 = no object


class PixelData:
    def __init__(self, **fields):
        self.__dict__.update(fields)


def _cls_row(label, strength=5.0):
    r = torch.zeros(C + 1)
    r[label] = strength
    return r


def build(queries):
    """queries: list of (label, strength, [(y0, y1, x0, x1, logit), ...]) -> (mask_cls [nq, C+1], mask_pred [nq, H, W])"""
    cls = [_cls_row(C - 1)]
    mp = [torch.full((H, W), -5.0)]
    for label, strength, regions in queries:
        cls.append(_cls_row(label, strength))
        m = torch.full((H, W), -20.0)
        for y0, y1, x0, x1, v in regions:
            m[y0:y1, x0:x1] = v
        mp.append(m)
    return torch.stack(cls), torch.stack(mp)


def designed():
    return [
        (0, 5.0, [(2, 6, 2, 6, 3.0)]),                          # 1: ties with 2 on its whole region, wins it (lower index)
        (0, 5.0, [(2, 6, 2, 14, 3.0)]),                         # 2: same class row: mask 32 / original 48
        (1, 5.0, [(10, 12, 0, 4, 2.0)]),                        # 3: loses 2 of its 8 pixels to 4: ratio exactly 0.75
        (1, 5.0, [(10, 12, 3, 7, 4.0)]),                        # 4
        (2, 5.0, [(14, 15, 0, 5, 2.0)]),                        # 5: loses 2 of 5 to 6: ratio 0.6
        (3, 5.0, [(14, 15, 3, 8, 4.0), (20, 22, 20, 24, 2.0)]),  # 6: stuff
        (3, 5.0, [(20, 22, 26, 30, 2.0)]),                      # 7: stuff of the same class: merged with 6
        (0, 5.0, [(16, 18, 16, 20, 1.0)]),                      # 8: dominated by 9 everywhere: mask 0, original 8
        (1, 5.0, [(16, 18, 16, 20, 3.0)]),                      # 9: takes the instance id 8 did not use
        (2, 5.0, [(0, 2, 20, 24, 0.0), (0, 2, 24, 28, -1e-8), (0, 2, 28, 30, -1e-6)]),  # 10: sigmoid exactly 0.5, then < 0.5
        (C, 6.0, [(20, 24, 0, 8, 6.0)]),                        # 11: argmax on the no-object class: not kept
        (2, 5.0, [(5, 10, 18, 32, -0.5), (6, 9, 20, 30, 0.5)]),  # 12: sigmoid < 0.5 on 40 of its 70 pixels
        (0, 2.5, [(18, 20, 8, 14, 2.0)]),                       # 13: weaker class score (object_mask_thr case)
    ]


def main():
    g = torch.Generator().manual_seed(4321)
    fh = load_defs("mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py", ["panoptic_postprocess"],
                   cls="MaskFormerFusionHead")
    fh.update(INSTANCE_OFFSET=1000, PixelData=PixelData)
    rf = load_defs("mmdet/rsprompter/models.py", ["predict"], cls="RSMaskFormerFusionHead")

    def head(cfg):
        self_ = SimpleNamespace(test_cfg=cfg, num_classes=C, num_things_classes=THINGS)
        self_.panoptic_postprocess = lambda c, m: fh["panoptic_postprocess"](self_, c, m)
        return self_

    mask_cls, mask_pred = build(designed())
    s13 = float(F.softmax(mask_cls[13], dim=-1).max())       # the exact fp32 score of query 13, as a Python float
    cases = dict(
        ties=dict(iou_thr=0.5),
        iou_exact=dict(iou_thr=0.75),
        filter_low_score=dict(iou_thr=0.75, filter_low_score=True),
        score_equals_thr=dict(iou_thr=0.75, object_mask_thr=s13),
        score_below_thr=dict(iou_thr=0.75, object_mask_thr=s13 - 1e-3),
        none_kept=dict(object_mask_thr=0.9999),
        defaults=dict(),
    )
    fx = dict(num_classes=C, num_things_classes=THINGS, mask_cls=mask_cls, mask_pred=mask_pred, cases={})
    for name, cfg in cases.items():
        fx["cases"][name] = dict(test_cfg=cfg, pan=fh["panoptic_postprocess"](head(cfg), mask_cls, mask_pred).sem_seg)

    # RSMaskFormerFusionHead.predict of a resized, padded image: ori 30 x 40, scale 1.5 -> 45 x 60 in a 48 x 64 batch;
    # low-res blob logits up-sampled to the batch shape as RSMask2FormerHead.predict does (M:652-656)
    nq, hm, wm = 12, 12, 16
    yy, xx = torch.meshgrid(torch.arange(hm, dtype=torch.float32), torch.arange(wm, dtype=torch.float32), indexing="ij")
    cy, cx = torch.rand(nq, 1, 1, generator=g) * hm, torch.rand(nq, 1, 1, generator=g) * wm
    rr = 1.5 + torch.rand(nq, 1, 1, generator=g) * 4
    low = (rr - ((yy - cy) ** 2 + (xx - cx) ** 2).sqrt()) * 1.7
    pcls = torch.randn(nq, C + 1, generator=g)
    pcls[torch.arange(nq), torch.randint(0, C, (nq,), generator=g)] += 6.0
    pcls[3, C] += 12.0                                            # one query on the no-object class
    up = F.interpolate(low[None], size=(48, 64), mode="bilinear", align_corners=False)
    meta = dict(img_shape=(45, 60), ori_shape=(30, 40), scale_factor=(1.5, 1.5), batch_input_shape=(48, 64))
    fx["predict"] = dict(mask_cls=pcls, logits=low, mask_pred=up[0], meta=meta, runs={})
    for rescale in (True, False):
        for flt in (False, True):
            cfg = dict(iou_thr=0.8, filter_low_score=flt, object_mask_thr=0.8)
            res = rf["predict"](head(cfg), pcls[None], up, [SimpleNamespace(metainfo=meta)], rescale=rescale)[0]
            assert set(res) == {"pan_results"}                  # panoptic_on defaults to True, instance_on to False
            fx["predict"]["runs"][(rescale, flt)] = dict(test_cfg=cfg, pan=res["pan_results"].sem_seg)

    torch.save(fx, OUT)
    print("wrote", OUT)
    for name, c in fx["cases"].items():
        print(name, torch.unique(c["pan"]).tolist())
    for k, c in fx["predict"]["runs"].items():
        print("predict", k, tuple(c["pan"].shape), torch.unique(c["pan"]).tolist())


if __name__ == "__main__":
    main()
