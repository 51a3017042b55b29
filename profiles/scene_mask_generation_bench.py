"""Segment-everything over whole scenes (rsprompter_b200.mask_generation.generate_scene_masks) on seeded synthetic
weights and scenes.

    python profiles/scene_mask_generation_bench.py [--archs base huge] [--sizes 4096 8192] [--repeats 1]
        [--thresholds hf_default zero zero_blobs] [--out r.json]

Workloads: ViT-B and ViT-H, seeded smooth uint8 scenes of 4096^2 and 8192^2 pixels on the device, 1024^2 windows at
the default overlap (25 and 121 windows) in batches of 4, the default 32 x 32 grid in calls of 64 prompts, with HF's
default thresholds, with every threshold 0 (every candidate reaches the crop-edge rule), and zero_blobs: thresholds 0
with the decoder's outputs replaced by seeded blob fields (_Blobs), because the seeded weights' masks each cover their
whole window, so the rule drops all of them and the RLE and merge stages would have nothing to do.  Per workload:

  * scene_ms: one whole generate_scene_masks call, host clock (it ends in host reads); tiles/s from it;
  * the split, each stage ended by a device synchronise and summed over the batches: tiles_ms (resize, encoder,
    decoder + crop stats, window NMS, paste), rle_ms (placed RLE of the kept masks into the scene), merge_ms (the
    cross-window NMS and its gathers);
  * candidates before and after the merge;
  * windows_ms: the same windows as independent generate_masks(output_rle_mask=True) calls on batches of 4 views of
    the scene, alternated with scene_ms in this process; scene_ms - windows_ms is the cost of scene mode (edge rule,
    placed RLE, merge).
Best of the repeats each.  The card's name and power limit are read in the same run.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

THRESHOLDS = {"hf_default": dict(pred_iou_thresh=0.88, stability_score_thresh=0.95),
              "zero": dict(pred_iou_thresh=0.0, stability_score_thresh=0.0),
              "zero_blobs": dict(pred_iou_thresh=0.0, stability_score_thresh=0.0)}


class _Blobs:
    """Decoder outputs in place of the seeded decoder's (whose masks all cover their window, so the edge rule drops
    every one): per prompt of a 32 x 32 grid, 3 fields each holding one Gaussian blob of seeded centre and radius, the
    same for every window, so windows keep masks and the RLE and merge stages have work."""

    def __init__(self, dev):
        g = torch.Generator().manual_seed(7)
        n = 1024 * 3
        cy, cx = torch.rand(n, generator=g) * 300 - 22, torch.rand(n, generator=g) * 300 - 22
        r = 4 + 40 * torch.rand(n, generator=g)
        yy, xx = torch.arange(256.0)[None, :, None], torch.arange(256.0)[None, None, :]
        low = torch.empty(n, 256, 256)
        for i in range(0, n, 256):
            d2 = (yy - cy[i:i + 256, None, None]) ** 2 + (xx - cx[i:i + 256, None, None]) ** 2
            low[i:i + 256] = 12 * torch.exp(-d2 / (2 * r[i:i + 256, None, None] ** 2)) - 4
        self.low = low.view(1024, 3, 256, 256).to(dev)
        self.iou = torch.rand(1024, 3, generator=g).to(dev)
        self.served = 0

    def __call__(self, emb_rows, pos_rows, sparse, hw, **kw):
        q0 = self.served % 1024
        self.served += sparse.shape[0]
        return self.low[q0:q0 + sparse.shape[0]], self.iou[q0:q0 + sparse.shape[0]]


BATCH = 4


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, limit = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=limit)


def _model(arch_name: str):
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch
    arch, darch = VISION_ARCHS[arch_name], SamDecoderArch()
    sd = {"shared_image_embedding.positional_embedding":
          synthetic.positional_embedding_state_dict(arch, 4)["positional_embedding"]}
    sd.update({"vision_encoder." + k: v for k, v in synthetic.vision_encoder_state_dict(arch, seed=1).items()})
    sd.update({"mask_decoder." + k: v for k, v in synthetic.mask_decoder_state_dict(darch, seed=2).items()})
    sd.update({"prompt_encoder." + k: v for k, v in synthetic.prompt_encoder_state_dict(darch, seed=3).items()})
    model = MODELS.build(dict(type="RSSamModel", hf_pretrain_name=f"facebook/sam-vit-{arch_name}"))
    model.sam_model.load_state_dict(sd, strict=True)
    return model.cuda().eval()


def _scene(side: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, side // 256, side // 256, generator=g) * 255, (side, side), mode="bilinear",
                         align_corners=False)[0]
    return (base + 20 * torch.rand(3, side, side, generator=g)).clamp(0, 255).to(torch.uint8).cuda()


def _sync_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


@torch.no_grad()
def _staged(model, scene, thr) -> dict:
    """generate_scene_masks' stages one by one, each ended by a synchronise."""
    from rsprompter_b200 import mask_generation as mg
    sam = model.sam_model
    H, W = int(scene.shape[1]), int(scene.shape[2])
    S = sam.varch.image_size
    crops = mg.scene_crop_boxes((H, W), S, 0.25)
    p = dict(points_per_side=32, points_per_batch=64, stability_score_offset=1.0, mask_threshold=0.0, **thr)
    t_tiles = t_rle = 0.0
    tiles = []
    for b0 in range(0, len(crops), BATCH):
        boxes = crops[b0:b0 + BATCH]

        def tile_stage():
            views = [scene[:, y0:y1, x0:x1] for x0, y0, x1, y1 in boxes]
            pix, sizes, reshaped = mg._inputs(sam, views, None, None, None, scene.device)
            cand = mg._candidates(sam, sam._encode(pix), sizes, reshaped, p, crops=[(cb, (H, W)) for cb in boxes])
            idx, counts, idx_host = mg._nms(cand["iou"], cand["keep"], cand["boxes"], 0.7)
            return mg._outputs(cand, idx, counts, idx_host, 0.0, S)
        out, ms = _sync_ms(tile_stage)
        t_tiles += ms
        _, ms = _sync_ms(lambda: mg._add_rle(out, places=[(H, W, y0, x0) for x0, y0, _, _ in boxes]))
        t_rle += ms
        for r in out:
            del r["masks"]
        tiles.extend(out)
    res, t_merge = _sync_ms(lambda: mg._merge_tiles(tiles, crops, (H, W), 0.7, scene.device))
    return dict(tiles_ms=t_tiles, rle_ms=t_rle, merge_ms=t_merge, windows=len(crops),
                before_merge=sum(r["scores"].shape[0] for r in tiles), after_merge=len(res["rle"]))


def _windows(model, scene, thr):
    from rsprompter_b200 import mask_generation as mg
    crops = mg.scene_crop_boxes(tuple(scene.shape[1:]), 1024, 0.25)
    for b0 in range(0, len(crops), BATCH):
        views = [scene[:, y0:y1, x0:x1] for x0, y0, x1, y1 in crops[b0:b0 + BATCH]]
        mg.generate_masks(model, views, output_rle_mask=True, **thr)


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser()
    ap.add_argument("--archs", nargs="+", default=["base", "huge"])
    ap.add_argument("--sizes", nargs="+", type=int, default=[4096, 8192])
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--thresholds", nargs="+", default=list(THRESHOLDS), choices=list(THRESHOLDS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    from rsprompter_b200 import mask_generation as mg
    card = _card()
    print(f"{card['gpu']}, power limit {card['power_limit']}", flush=True)
    rows = []
    for arch in args.archs:
        model = _model(arch)
        warm = _scene(2048, 0)
        for thr in list(THRESHOLDS.values())[:2]:     # every shape and code path once
            mg.generate_scene_masks(model, warm, **thr)
            _windows(model, warm, thr)
        for side in args.sizes:
            scene = _scene(side, side)
            for name in args.thresholds:
                thr = THRESHOLDS[name]
                dec = model.sam_model.mask_decoder
                if name.endswith("_blobs"):
                    dec.decode = _Blobs(scene.device)
                elif "decode" in vars(dec):
                    del dec.decode
                best = dict(scene_ms=float("inf"), windows_ms=float("inf"))
                for _ in range(args.repeats):
                    _, ms = _sync_ms(lambda: mg.generate_scene_masks(model, scene, **thr))
                    best["scene_ms"] = min(best["scene_ms"], ms)
                    _, ms = _sync_ms(lambda: _windows(model, scene, thr))
                    best["windows_ms"] = min(best["windows_ms"], ms)
                st = _staged(model, scene, thr)
                row = dict(arch=arch, scene=side, thresholds=name, **st, **best,
                           tiles_per_s=st["windows"] / best["scene_ms"] * 1e3,
                           scene_mode_cost_ms=best["scene_ms"] - best["windows_ms"])
                print(json.dumps({k: round(v, 1) if isinstance(v, float) else v for k, v in row.items()}), flush=True)
                rows.append(row)
                torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    result = dict(card, rows=rows)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    return result


if __name__ == "__main__":
    main()
