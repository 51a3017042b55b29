"""Coarse layers of segment-everything over whole scenes: the antialiased resize kernel alone, and
generate_scene_masks(coarse_patch_sizes=...) on seeded synthetic weights and scenes.

    python profiles/scene_layers_bench.py [--archs base huge] [--sizes 4096 8192] [--workloads hf_default blobs]
        [--out r.json]

Part 1, rsp_resize_aa_pad_u8 against rsp_resize_pad_u8 (cv2 INTER_LINEAR) on the same views, and against torchvision's
CPU resize (tvF.resize(uint8, antialias=True), the one SamImageProcessor runs) of the same image: an 8192^2 and a
20 000 x 12 000 scene and a 1500 x 900 image, each to longest side 1024.  CUDA events over 20 launches after 3 warm-up
launches; bytes moved = the source read once + the horizontal-pass workspace written and read + the fp32 output.

Part 2, generate_scene_masks on 4096^2 and 8192^2 seeded scenes on the device, ViT-B and ViT-H, 1024^2 base windows
at overlap 0.25 in batches of 4, a 32 x 32 grid in calls of 64 prompts; workloads hf_default (HF's default thresholds)
and blobs (thresholds 0, the decoder's outputs replaced by scene_mask_generation_bench's seeded one-blob fields).
coarse_patch_sizes (), (4096,), (max(H, W),) and (4096, max(H, W)) alternate in one process (at 4096^2 only () and
(4096,), the whole scene).  Per call: the host clock around the call (it ends in host reads); then the same
call again with the stages wrapped, each ended by a device synchronise (resize, encoder, decoder + stats, window NMS,
outputs = paste + clean + RLE, merges).  The card's name and power limit are read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from scene_mask_generation_bench import THRESHOLDS, _Blobs, _card, _model, _scene  # noqa: E402

MEAN = tuple(255.0 * m for m in (0.485, 0.456, 0.406))
STD = tuple(255.0 * s for s in (0.229, 0.224, 0.225))


def _events_ms(fn, n=20, warm=3) -> float:
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def resize_part() -> list:
    from torchvision.transforms.v2 import functional as tvF

    from rsprompter_b200 import _lib
    from rsprompter_b200.mask_generation import preprocess_shape
    rows = []
    for H, W in ((8192, 8192), (12000, 20000), (1500, 900)):
        g = torch.Generator().manual_seed(H + W)
        img = torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8)
        dev = img.cuda()
        nh, nw = preprocess_shape((H, W), 1024)
        out = torch.empty(1, 3, 1024, 1024, device="cuda")
        aa = _events_ms(lambda: _lib.resize_aa_pad_u8([dev], [(nh, nw)], out, MEAN, STD, False, MEAN))
        cv = _events_ms(lambda: _lib.resize_pad_u8([dev], [(nh, nw)], out, MEAN, STD, False, MEAN))
        t = time.perf_counter()
        tvF.resize(img, [nh, nw], interpolation=tvF.InterpolationMode.BILINEAR, antialias=True)
        cpu = (time.perf_counter() - t) * 1e3
        moved = 3 * H * W + 2 * 3 * H * nw + 3 * 1024 * 1024 * 4
        rows.append(dict(what=f"{H} x {W} -> {nh} x {nw}", aa_ms=round(aa, 3), aa_GBps=round(moved / aa / 1e6, 1),
                         cv2_linear_ms=round(cv, 3), torchvision_cpu_ms=round(cpu, 1), bytes_moved=moved))
        print(json.dumps(rows[-1]), flush=True)
        del dev
    return rows


STAGES = ("_inputs", "_candidates", "_nms", "_outputs", "_remove_small_regions", "_add_rle", "_coarse_outputs",
          "_merge_tiles", "_merge_layers")


def _staged(fn) -> dict:
    """fn() with each stage of mask_generation wrapped in device synchronises; -> ms per stage, summed."""
    from rsprompter_b200 import mask_generation as mg
    times = dict.fromkeys(STAGES, 0.0)
    saved = {k: getattr(mg, k) for k in STAGES}

    def wrap(name, f):
        def g(*a, **kw):
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = f(*a, **kw)
            torch.cuda.synchronize()
            times[name] += (time.perf_counter() - t) * 1e3
            return r
        return g
    for k in STAGES:
        setattr(mg, k, wrap(k, saved[k]))
    try:
        fn()
    finally:
        for k in STAGES:
            setattr(mg, k, saved[k])
    return {k: round(v, 1) for k, v in times.items() if v}


@torch.no_grad()
def layers_part(archs, sizes, workloads) -> list:
    from rsprompter_b200 import mask_generation as mg
    rows = []
    for arch in archs:
        model = _model(arch)
        dec = model.sam_model.mask_decoder
        for side in sizes:
            scene = _scene(side, seed=side)
            configs = [(), (4096,), (side,), (4096, side)] if side > 4096 else [(), (4096,)]
            for wl in workloads:
                thr = THRESHOLDS["zero_blobs" if wl == "blobs" else wl]
                kw = dict(points_per_side=32, points_per_batch=64, batch_size=4, **thr)
                if wl == "blobs":
                    dec.decode = _Blobs(scene.device)
                for coarse in configs:
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    res = mg.generate_scene_masks(model, scene, coarse_patch_sizes=coarse, **kw)
                    torch.cuda.synchronize()
                    ms = (time.perf_counter() - t) * 1e3
                    stages = _staged(lambda: mg.generate_scene_masks(model, scene, coarse_patch_sizes=coarse, **kw))
                    layers = res["layers"].bincount(minlength=len(coarse) + 1).tolist()
                    rows.append(dict(arch=arch, scene=side, workload=wl, coarse=list(coarse), call_ms=round(ms, 1),
                                     kept_per_layer=layers, stages_ms=stages))
                    print(json.dumps(rows[-1]), flush=True)
                    del res
                if wl == "blobs":
                    del dec.decode
            del scene
        del model, dec
        torch.cuda.empty_cache()
    return rows


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser()
    ap.add_argument("--archs", nargs="+", default=["base", "huge"])
    ap.add_argument("--sizes", nargs="+", type=int, default=[4096, 8192])
    ap.add_argument("--workloads", nargs="+", default=["hf_default", "blobs"])
    ap.add_argument("--skip-resize", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    res = dict(card=_card())
    print(json.dumps(res), flush=True)
    if not args.skip_resize:
        res["resize"] = resize_part()
    res["layers"] = layers_part(args.archs, args.sizes, args.workloads)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
