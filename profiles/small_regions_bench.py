"""Small-region removal of segment-everything (SAM's min_mask_region_area) on the GPU against SAM's host loop.

    python profiles/small_regions_bench.py [--counts 100 300] [--area 100] [--out result.json]

Workloads: n = 100 and 300 bit-packed masks of 1024 x 1024 (the kept masks of a call are of that order), two kinds:
"blob" (a smoothed random field, thresholded: SAM-like regions with a few holes and crumbs) and "noise"
(salt-and-pepper at density 0.5, near the 8-connected percolation point: the most components and the longest union
chains).  Per workload:

  * kernel_ms: rsp_mask_small_regions_bits in holes mode then islands mode over all n masks, the way generate_masks
    calls it, CUDA events around 10 repeats after a warm-up, mean;
  * floor_us: bytes the two calls must move at least (each reads the bits 5 times and writes them once, and makes 5
    passes over 4-byte labels per 2 x 2 block) over the data sheet's 3.35 TB/s: a bound from shapes, not a time;
  * host_ms: SAM's loop (remove_small_regions holes then islands per mask, cv2.connectedComponentsWithStats, as the
    oracle restates it) over the same masks, from unpacked bool arrays, host clock; cv2's thread count is printed.

Then the whole generate_masks call (ViT-B, seeded synthetic weights, one 1024 x 1024 image, the default 32 x 32 grid,
filters off) with min_mask_region_area 0 and --area, host clock, best of 3 each, alternated.

The card's name and power limit are printed with the numbers.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HW = 1024
HBM_BYTES_PER_S = 3.35e12


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, limit = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=limit)


def _masks(kind: str, n: int, seed: int) -> torch.Tensor:
    """bool [n, HW, HW] on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "noise":
        return torch.rand(n, HW, HW, generator=g, device="cuda") < 0.5
    out = torch.empty(n, HW, HW, dtype=torch.bool, device="cuda")
    for i in range(n):
        f = F.interpolate(torch.randn(1, 1, 12, 12, generator=g, device="cuda"), (HW, HW), mode="bilinear",
                          align_corners=False)
        f = f + 0.35 * F.interpolate(torch.randn(1, 1, 160, 160, generator=g, device="cuda"), (HW, HW),
                                     mode="bilinear", align_corners=False)
        out[i] = f[0, 0] > 0.5
    return out


def _kernel_ms(bits: torch.Tensor, area: int, reps: int = 10) -> float:
    from rsprompter_b200 import _lib
    n, H, _ = bits.shape
    ws = torch.empty(_lib.small_regions_ws_bytes(n, H, HW), device="cuda", dtype=torch.uint8)
    tmp, out = torch.empty_like(bits), torch.empty_like(bits)

    def run():
        _lib.mask_small_regions_bits(bits, HW, area, "holes", out=tmp, ws=ws)
        _lib.mask_small_regions_bits(tmp, HW, area, "islands", out=out, ws=ws)

    run()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        run()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def _floor_us(n: int) -> float:
    bits = n * HW * HW / 8
    labels = n * (HW // 2) * (HW // 2) * 4
    return 2 * (6 * bits + 5 * labels) / HBM_BYTES_PER_S * 1e6


def _host_ms(masks: np.ndarray, area: float) -> tuple:
    from oracle.restate_small_regions import remove_small_regions
    t = time.perf_counter()
    marks = []
    for i, m in enumerate(masks):
        m, _ = remove_small_regions(m, area, "holes")
        remove_small_regions(m, area, "islands")
        marks.append(time.perf_counter() - t)
    return [1e3 * x for x in marks]


def _model():
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch
    arch, darch = VISION_ARCHS["base"], SamDecoderArch()
    sd = {"shared_image_embedding.positional_embedding":
          synthetic.positional_embedding_state_dict(arch, 4)["positional_embedding"]}
    sd.update({"vision_encoder." + k: v for k, v in synthetic.vision_encoder_state_dict(arch, seed=1).items()})
    sd.update({"mask_decoder." + k: v for k, v in synthetic.mask_decoder_state_dict(darch, seed=2).items()})
    sd.update({"prompt_encoder." + k: v for k, v in synthetic.prompt_encoder_state_dict(darch, seed=3).items()})
    model = MODELS.build(dict(type="RSSamModel", hf_pretrain_name="facebook/sam-vit-base"))
    model.sam_model.load_state_dict(sd, strict=True)
    return model.cuda().eval()


def _call_ms(model, img, area: float, repeats: int = 3) -> dict:
    times, kept = {0.0: [], area: []}, {}
    for _ in range(repeats + 1):
        for a in (0.0, area):
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = model.generate_masks(img, pred_iou_thresh=0.0, stability_score_thresh=0.0, min_mask_region_area=a,
                                     output_rle_mask=True)[0]
            torch.cuda.synchronize()
            times[a].append(1e3 * (time.perf_counter() - t))
            kept[a] = int(r["masks"].shape[0])
    return {f"call_ms_area_{a:g}": min(ts[1:]) for a, ts in times.items()} | \
           {f"kept_area_{a:g}": k for a, k in kept.items()}


def main() -> None:
    import cv2

    from rsprompter_b200 import _lib
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--counts", nargs="+", type=int, default=[100, 300])
    ap.add_argument("--area", type=float, default=100.0)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = _card()
    print(f"{card['gpu']}, power limit {card['power_limit']}, cv2 threads {cv2.getNumThreads()}", flush=True)
    rows = []
    area = int(np.ceil(args.area))
    for kind in ("blob", "noise"):
        masks = _masks(kind, max(args.counts), seed=1)
        bits = _lib.pack_mask_bits(masks)
        host = _host_ms(masks.cpu().numpy(), args.area)
        for n in args.counts:
            row = dict(kind=kind, n=n, kernel_ms=round(_kernel_ms(bits[:n].contiguous(), area), 3),
                       floor_us=round(_floor_us(n), 1), host_ms=round(host[n - 1], 1))
            print(json.dumps(row), flush=True)
            rows.append(row)
        del masks, bits
    g = torch.Generator().manual_seed(0)
    img = F.interpolate(torch.rand(1, 3, 8, 8, generator=g) * 255, (HW, HW), mode="bilinear", align_corners=False)[0]
    img = (img + 20 * torch.rand(3, HW, HW, generator=g)).clamp(0, 255).to(torch.uint8)
    call = _call_ms(_model(), img, args.area)
    print(json.dumps(call), flush=True)
    res = dict(card, area=args.area, cv2_threads=cv2.getNumThreads(), kernels=rows, generate_masks=call)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
