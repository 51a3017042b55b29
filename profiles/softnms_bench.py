"""Soft-NMS (rsp_soft_nms_batched) against the hard NMS it sits beside, on seeded inputs.

    python profiles/softnms_bench.py [--repeats 20]

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * roi_head: the kernel alone on the RoI head's problem (B = 8 images, 1000 RoIs x C classes, max_keep 100, candidates
    in (RoI, class) order) against rsp_nms_batched + rsp_compact_keep (with the score sort they need) on the same
    candidates, C in {1, 10};
  * anchor_step: one RSPrompterAnchor ViT-B predict_records step (8 images of 1024^2, CUDA graphs on, seeded random
    weights) with rcnn.nms soft against hard;
  * merge: merge_tile_records over 25, 121 and 441 tiles of 100 slots (2 500, 12 100, 44 100 candidates, 10 labels,
    seeded boxes), soft against hard;
  * restatement: the literal Python loop of oracle.restate_soft_nms on one CPU core at 1 000 candidates (the
    restatement, not mmcv's C++).
Device times are CUDA events over ``--repeats`` calls after two warm-up calls.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    name, power = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power)


def _time(fn, repeats: int) -> float:
    """ms per call, CUDA events."""
    fn(); fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeats


def _candidates(B, R, C, seed):
    g = torch.Generator().manual_seed(seed)
    ctr = torch.rand(B, R, 1, 2, generator=g) * 1024
    wh = torch.exp(torch.rand(B, R, 1, 2, generator=g) * 4 + 2)
    jit = torch.randn(B, R, C, 4, generator=g) * 4
    boxes = (torch.cat([ctr - wh / 2, ctr + wh / 2], -1) + jit).clamp(0, 1024).reshape(B, R * C, 4)
    scores = torch.rand(B, R * C, generator=g)
    labels = torch.arange(C).repeat(R).view(1, -1).expand(B, -1).contiguous()
    return boxes.cuda().contiguous(), scores.cuda().contiguous(), labels.cuda()


def bench_roi(card, repeats):
    from rsprompter_b200 import _lib
    for C in (1, 10):
        boxes, scores, labels = _candidates(8, 1000, C, C)
        nv = torch.full((8,), 1000 * C, dtype=torch.int32, device="cuda")

        def soft():
            return _lib.soft_nms_batched(boxes, scores, labels, nv, C, 0.5, 0.5, 0.05, "linear", K=100)

        def hard():
            s, o = torch.sort(scores, dim=1, descending=True, stable=True)
            b = torch.gather(boxes, 1, o[:, :, None].expand(-1, -1, 4)).contiguous()
            lab = torch.gather(labels, 1, o).contiguous()
            keep = _lib.nms_batched(b, lab, nv, 0.5, max_keep=100)
            return _lib.compact_keep(keep, b, s.contiguous(), lab, 100)
        print(json.dumps(dict(card, case="roi_head", B=8, rois=1000, classes=C, max_keep=100,
                              soft_ms=round(_time(soft, repeats), 4), hard_ms=round(_time(hard, repeats), 4))),
              flush=True)


def bench_anchor(card, repeats):
    from rsprompter_b200 import model_configs, synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS
    sd = synthetic.anchor_detector_state_dict(VISION_ARCHS["base"], 10, len(SELECT_LAYERS["base"]), seed=0)
    x = (torch.randn(8, 3, 1024, 1024, generator=torch.Generator().manual_seed(1)) * 50).cuda()
    out = {}
    for typ in ("nms", "soft_nms"):
        cfg = model_configs.anchor_model_cfg("base", 10)
        if typ == "soft_nms":
            cfg["test_cfg"]["rcnn"]["nms"] = dict(type="soft_nms", iou_threshold=0.5, min_score=0.05)
        m = MODELS.build(cfg)
        m.load_state_dict(sd)
        m = m.cuda().enable_cuda_graphs()
        out[typ] = _time(lambda: m.predict_records(x), max(3, repeats // 4))
        del m
        torch.cuda.empty_cache()
    print(json.dumps(dict(card, case="anchor_step", arch="vit-b", images=8, cuda_graphs=True,
                          soft_ms=round(out["soft_nms"], 3), hard_ms=round(out["nms"], 3))), flush=True)


def bench_merge(card, repeats):
    from rsprompter_b200.large_image import merge_tile_records
    from rsprompter_b200.results import ResultRecord
    P, M = 1024, 100
    for side in (5, 11, 21):
        n_tiles = side * side
        g = torch.Generator().manual_seed(side)
        recs, origins = [], []
        step = 768
        org = [(x * step, y * step) for y in range(side) for x in range(side)]
        for i in range(0, n_tiles, 8):
            chunk = org[i:i + 8]
            rec = ResultRecord(8, M, (P, P), device="cuda")
            xy = torch.rand(8, M, 2, generator=g) * (P - 8)
            wh = 4 + torch.rand(8, M, 2, generator=g) * 120
            b = torch.cat([xy, torch.minimum(xy + wh, torch.full_like(xy, float(P)))], 2)
            s = torch.rand(8, M, 1, generator=g)
            lab = torch.randint(0, 10, (8, M, 1), generator=g).float()
            rec.rows.copy_(torch.cat([b, s, lab], 2))
            rec.counts.fill_(M)
            recs.append(rec)
            origins.append(chunk)
        hw = (step * (side - 1) + P, step * (side - 1) + P)
        r = {}
        for typ in ("nms", "soft_nms"):
            def run(typ=typ):
                return merge_tile_records(recs, origins, hw, merge_iou_thr=0.25, nms_type=typ)
            run()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            reps = max(2, repeats // 4)
            for _ in range(reps):
                kept = run()
            r[typ] = ((time.perf_counter() - t0) / reps * 1e3, int(kept["bboxes"].shape[0]))
        print(json.dumps(dict(card, case="merge", tiles=n_tiles, candidates=n_tiles * M,
                              soft_ms=round(r["soft_nms"][0], 3), soft_kept=r["soft_nms"][1],
                              hard_ms=round(r["nms"][0], 3), hard_kept=r["nms"][1])), flush=True)


def bench_restatement(card):
    from oracle.restate_soft_nms import soft_nms_literal
    boxes, scores, _ = _candidates(1, 1000, 1, 5)
    b, s = boxes[0].cpu().numpy(), scores[0].cpu().numpy()
    t0 = time.process_time()
    soft_nms_literal(b, s, 0.5, 0.5, 0.05, "linear")
    print(json.dumps(dict(card, case="restatement_literal_python_1core", candidates=1000,
                          ms=round((time.process_time() - t0) * 1e3, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "softnms_bench needs a GPU"
    card = _card()
    bench_roi(card, args.repeats)
    bench_merge(card, args.repeats)
    bench_anchor(card, args.repeats)
    bench_restatement(card)


if __name__ == "__main__":
    main()
