"""Panoptic post-processing of the query detectors on the GPU against the reference's torch loop, same GPU.

    python profiles/panoptic_bench.py [--steps 20] [--out result.json]

Workloads (the C3 shapes: bs 8, 100 queries, 256 x 256 mask logits, 1024 x 1024 batch), each with 10 / 50 / 100 kept
queries (the class logits make exactly that many queries pass object_mask_thr 0.8):
  * batch: every image at the batch shape (one bilinear x4 resize);
  * nwpu: an NWPU-like resized mix, ori_shape 800 x 1000 / 700 x 933 / 600 x 800 / 1024 x 1024 repeated, resized to a
    1024 long side and padded (resize to the batch shape, crop, resize to ori_shape, with rescale=True).
The mask logits are seeded blob fields (one steep blob per query over a flat background query), so no pixel sits within
2^-20 of a tie and both paths must give the same maps; the script checks that every map is equal.

  * ours_ms: RSMaskFormerFusionHead.panoptic_postprocess_batched from the low-res logits (softmax, keep, the three
    kernels per launch group);
  * ref_ms: the reference's path on the same GPU in torch: F.interpolate of all queries to the batch shape
    (M:652-656), per image the crop / rescale (M:679-691) and MaskFormerFusionHead.panoptic_postprocess
    (maskformer_fusion_head.py:41-106, restated in oracle/restate_panoptic.py: two .item() host reads per kept query).
CUDA events around --steps calls after a warm-up, the two paths alternated in one process; mean per batch.
The card's name and power limit are printed with the numbers.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, NQ, HM, BATCH = 8, 100, 256, (1024, 1024)
C, THINGS = 10, 10
NWPU = [(800, 1000), (700, 933), (600, 800), (1024, 1024)]


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, limit = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=limit)


def _inputs(kept: int, seed: int):
    g = torch.Generator(device="cuda").manual_seed(seed)
    cls = torch.randn(B, NQ, C + 1, generator=g, device="cuda") * 0.3
    lab = torch.randint(0, C, (B, NQ), generator=g, device="cuda")
    strong = torch.zeros(B, NQ, dtype=torch.bool, device="cuda")
    strong[:, :kept] = True
    cls.scatter_add_(2, lab[..., None], torch.where(strong, 8.0, 0.0)[..., None])
    yy, xx = torch.meshgrid(torch.arange(HM, device="cuda", dtype=torch.float32),
                            torch.arange(HM, device="cuda", dtype=torch.float32), indexing="ij")
    cy = torch.rand(B * NQ, 1, 1, generator=g, device="cuda") * HM
    cx = torch.rand(B * NQ, 1, 1, generator=g, device="cuda") * HM
    r = 4 + torch.rand(B * NQ, 1, 1, generator=g, device="cuda") * 40
    logits = ((r - ((yy - cy) ** 2 + (xx - cx) ** 2).sqrt()) * 40).clamp(min=-30.0)
    logits[::NQ] = -2.0                    # query 0 of each image: a flat background
    return cls, logits.contiguous()


def _metas(kind: str):
    if kind == "batch":
        return None
    out = []
    for i in range(B):
        ori = NWPU[i % len(NWPU)]
        s = min(BATCH[0] / ori[0], BATCH[1] / ori[1])
        new = (int(ori[0] * s + 0.5), int(ori[1] * s + 0.5))
        sf = (new[1] / ori[1], new[0] / ori[0])
        crop = (min(int(ori[0] * sf[1]), BATCH[0]), min(int(ori[1] * sf[0]), BATCH[1]))
        out.append(None if ori == BATCH else dict(ori_hw=ori, crop_hw=crop, scale_factor=sf))
    return out


def _reference(cls, logits, metas, cfg):
    from oracle import restate_panoptic as rp
    up = F.interpolate(logits.view(B, NQ, HM, HM), size=BATCH, mode="bilinear", align_corners=False)
    out = []
    for b in range(B):
        mp = up[b]
        m = None if metas is None else metas[b]
        if m is not None:
            mp = mp[:, :m["crop_hw"][0], :m["crop_hw"][1]]
            mp = F.interpolate(mp[:, None], size=m["ori_hw"], mode="bilinear", align_corners=False)[:, 0]
        out.append(rp.panoptic_postprocess(cls[b], mp, C, THINGS, cfg))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "panoptic_bench needs a GPU"
    from rsprompter_b200.registry import MODELS
    cfg = dict(object_mask_thr=0.8, iou_thr=0.8)
    head = MODELS.build(dict(type="RSMaskFormerFusionHead", num_things_classes=THINGS, num_stuff_classes=0,
                             test_cfg=cfg))
    res = dict(card=_card(), batch=B, queries=NQ, logits=HM, out=BATCH, steps=a.steps, rows=[])
    print(json.dumps(res["card"]))
    for kind in ("batch", "nwpu"):
        metas = _metas(kind)
        for kept in (10, 50, 100):
            cls, logits = _inputs(kept, seed=kept)
            ours = lambda: head.panoptic_postprocess_batched(cls, logits, BATCH, metas=metas)[0]  # noqa: E731
            ref = lambda: _reference(cls, logits, metas, cfg)  # noqa: E731
            got, exp = ours(), ref()
            equal = all(torch.equal(x, y) for x, y in zip(got, exp))
            n_kept = int((torch.softmax(cls, -1).max(-1).values > 0.8).sum().item()) // B
            t = {"ours": 0.0, "ref": 0.0}
            for _ in range(2):
                ours(), ref()
            for _ in range(a.steps):
                for name, fn in (("ours", ours), ("ref", ref)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    t[name] += e0.elapsed_time(e1)
            row = dict(workload=kind, kept=n_kept, ours_ms=t["ours"] / a.steps, ref_ms=t["ref"] / a.steps,
                       equal=equal, segments=int(sum(len(torch.unique(x)) for x in got)))
            row["speedup"] = row["ref_ms"] / row["ours_ms"]
            res["rows"].append(row)
            print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
