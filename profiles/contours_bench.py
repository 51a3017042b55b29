"""Mask polygons on the GPU (_lib.mask_contours, csrc/contours.cu) against the reference path on the same masks:
copy the masks to the host, then mmdet's bitmap_to_polygon (cv2.findContours(RETR_CCOMP, CHAIN_APPROX_NONE)) per
mask.  Both are timed by host clock around work that ends in a device synchronise (the GPU call synchronises twice
itself), alternated in one process after a warm-up.  The device half of the GPU call (both passes and the read of the
totals between them, without the copy and the per-contour numpy arrays) is timed with CUDA events over repeated
calls.  The card's name and power limit are read in the same run.

    python profiles/contours_bench.py [--reps 3] [--out contours_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rsprompter_b200 import _lib  # noqa: E402


def _blobs(n, hw, seed):
    g = torch.Generator().manual_seed(seed)
    f = F.interpolate(torch.randn(n, 1, hw // 32, hw // 32, generator=g), (hw, hw), mode="bilinear",
                      align_corners=False)[:, 0]
    return f > 0.8


def _noise(n, hw, seed):
    return torch.rand(n, hw, hw, generator=torch.Generator().manual_seed(seed)) < 0.5


def _canvases(bits, W):
    n, H, ld = bits.shape
    return [(H, W, [(0, j * H * ld, ld, H, H, W, 0, 0)]) for j in range(n)]


def _gpu(bits, W):
    """The whole call: both passes, both host synchronisations, the copy and the per-contour numpy arrays."""
    return _lib.mask_contours([bits], _canvases(bits, W), _lib.CHAIN_APPROX_NONE)


def _device_fn(bits, W):
    """The device half alone (the two passes and the host read of the totals between them)."""
    n, H, ld = bits.shape
    rows = [(H, W, j, 1) for j in range(n)]
    parts_host = torch.tensor([(j * H * ld, ld, H, H, W, 0, 0) for j in range(n)], dtype=torch.int64).pin_memory()
    parts_d = parts_host.to(bits.device)
    return lambda: _lib._contours_device(bits.data_ptr(), rows, parts_d, parts_host, _lib.CHAIN_APPROX_NONE,
                                         bits.device)


def _reference(masks):
    host = masks.cpu().numpy()                         # device -> host copy of the masks
    out = []
    for m in host:
        outs = cv2.findContours(m.astype(np.uint8), cv2.RETR_CCOMP, cv2.CHAIN_APPROX_NONE)
        out.append(([c.reshape(-1, 2) for c in outs[-2]], outs[-1]))
    return out


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)
    ys, xs = torch.meshgrid(torch.arange(1024), torch.arange(1024), indexing="ij")
    serp = (ys % 4 == 0) | (xs == torch.where((ys // 4) % 2 == 0, 1023, 0))    # one border of about 0.5 M points
    cases = [("100 blob 1024^2", _blobs(100, 1024, 1)), ("300 blob 1024^2", _blobs(300, 1024, 2)),
             ("record 8 x 100 slots 1024^2", _blobs(800, 1024, 5)),
             ("100 noise 1024^2", _noise(100, 1024, 3)),     # the reference path takes over 2 minutes here
             ("4 serpentine 1024^2", serp[None].expand(4, -1, -1).contiguous())]
    rows = []
    for name, masks in cases:
        masks = masks.cuda()
        bits = _lib.pack_mask_bits(masks)
        W = masks.shape[-1]
        got = _gpu(bits, W)                            # warm-up, and the outputs agree (first masks)
        want = _reference(masks[:4])
        assert all(len(g[0]) == len(w[0]) and all(np.array_equal(x, y) for x, y in zip(g[0], w[0]))
                   for g, w in zip(got, want)), name
        dev = _device_fn(bits, W)
        dev()
        gpu_ms, ref_ms = [], []
        for _ in range(args.reps):                     # alternated
            gpu_ms.append(_time(lambda: _gpu(bits, W), 1))
            ref_ms.append(_time(lambda: _reference(masks), 1))
        row = dict(case=name, masks=int(masks.shape[0]), contours=sum(len(g[0]) for g in got),
                   points=int(sum(sum(len(c) for c in g[0]) for g in got)), device_ms=_events(dev, args.reps),
                   gpu_ms=float(np.median(gpu_ms)), reference_ms=float(np.median(ref_ms)))
        row["speedup"] = row["reference_ms"] / row["gpu_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        if args.out:
            with open(args.out, "w") as f:
                json.dump(dict(card=card, rows=rows), f, indent=1)
        del masks, bits, got, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
