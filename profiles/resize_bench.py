"""Timings of the device Resize + Pad (rsp_resize_pad_u8) against the host pipeline it replaces, and of large-scene
tiles at a resized patch size.  Prints one JSON line per measurement, each with the card name and power limit.

  * kernel: CUDA-event time per launch over >= 200 launches, bs 8 of 512^2 -> 1024^2 and a seeded mix of
    NWPU-like sizes (arbitrary sizes well below 1024^2);
  * host: cv2.resize(float32, INTER_LINEAR) + pad + HWC -> CHW of the same images on this machine's CPU, one core;
  * tiles/s of an 8192^2 scene through predict_large_image at patch 640 against patch 1024 (synthetic ViT-B
    anchor detector at 1024^2).

python profiles/resize_bench.py [--iters 200] [--skip-scene]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MEAN = [123.675, 116.28, 103.53]
STD = [58.395, 57.12, 57.375]
PAD = (0.406 * 255, 0.456 * 255, 0.485 * 255)


def _card() -> dict:
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return dict(card=name, power_limit_w=pl)


def _images(kind: str):
    g = np.random.default_rng(0)
    if kind == "512":
        hws = [(512, 512)] * 8
    else:   # NWPU VHR-10-like: assorted sizes, longest side 500-1000
        hws = [(int(g.integers(400, 900)), int(g.integers(500, 1000))) for _ in range(8)]
    return [g.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in hws]


def bench_kernel(kind: str, iters: int, card: dict) -> dict:
    from rsprompter_b200 import _lib
    from rsprompter_b200.preprocess import rescale_size
    imgs = _images(kind)
    dev = [torch.from_numpy(im).cuda().permute(2, 0, 1).contiguous() for im in imgs]
    sizes = [rescale_size(im.shape[:2], (1024, 1024)) for im in imgs]
    out = torch.empty(len(imgs), 3, 1024, 1024, device="cuda")
    for _ in range(10):
        _lib.resize_pad_u8(dev, sizes, out, MEAN, STD, True, PAD)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        _lib.resize_pad_u8(dev, sizes, out, MEAN, STD, True, PAD)
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / iters
    return dict(what=f"rsp_resize_pad_u8 bs8 {kind} -> 1024^2", ms_per_launch=round(ms, 4),
                note="includes the per-launch descriptor upload", **card)


def bench_host(kind: str, card: dict) -> dict:
    import cv2
    from rsprompter_b200.preprocess import rescale_size
    cv2.setNumThreads(1)
    imgs = _images(kind)
    reps = 3
    t0 = time.perf_counter()
    for _ in range(reps):
        for im in imgs:
            nh, nw = rescale_size(im.shape[:2], (1024, 1024))
            r = cv2.resize(im.astype(np.float32), (nw, nh), interpolation=cv2.INTER_LINEAR)
            p = np.empty((1024, 1024, 3), np.float32)
            p[...] = PAD
            p[:nh, :nw] = r
            np.ascontiguousarray(p.transpose(2, 0, 1))
    ms = (time.perf_counter() - t0) * 1e3 / reps
    return dict(what=f"host cv2.resize + pad + transpose bs8 {kind} -> 1024^2", ms_per_batch=round(ms, 2),
                cpu=os.uname().machine, threads=1, **card)


def bench_scene(card: dict) -> list:
    from rsprompter_b200 import model_configs, synthetic
    from rsprompter_b200.large_image import predict_large_image, slice_origins
    from rsprompter_b200.registry import MODELS
    cfg = model_configs.anchor_model_cfg("base", 10, mmpretrain_img_size=1024)
    cfg = dict(cfg, data_preprocessor=dict(type="DetDataPreprocessor", mean=MEAN, std=STD, bgr_to_rgb=True,
                                           pad_size_divisor=32))
    m = MODELS.build(cfg)
    m.load_state_dict(synthetic.anchor_detector_state_dict(m.backbone.vision_encoder.arch, 10, 0, seed=3,
                                                           pseudo_neck=True), strict=True)
    m = m.cuda().eval().enable_cuda_graphs()
    scene = np.random.default_rng(1).integers(0, 256, (8192, 8192, 3), dtype=np.uint8)
    scene_dev = torch.from_numpy(scene).cuda()
    out = []
    for P in (1024, 640):
        n = len(slice_origins((8192, 8192), P, 0.25))
        predict_large_image(m, scene_dev, patch_size=P)          # capture
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        predict_large_image(m, scene_dev, patch_size=P)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        out.append(dict(what=f"8192^2 scene, patch {P}, ViT-B anchor at 1024^2, bs 8, CUDA graphs", tiles=n,
                        seconds=round(s, 3), tiles_per_s=round(n / s, 2), **card))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--skip-scene", action="store_true")
    args = ap.parse_args()
    card = _card()
    rows = [bench_kernel("512", args.iters, card), bench_kernel("nwpu", args.iters, card)]
    try:
        rows += [bench_host("512", card), bench_host("nwpu", card)]
    except ImportError:
        rows.append(dict(what="host cv2 pipeline", note="cv2 not installed: not measured"))
    if not args.skip_scene:
        rows += bench_scene(card)
    for r in rows:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
