"""COCO RLE of one C3-sized batch of predicted masks (8 images x 100 instances at 1024^2): the device encoder
(rsp_mask_rle_*) against the host path it replaces (.cpu() + results.mask_to_coco_rle, one CPU core).

    python profiles/rle_bench.py [--iters 20] [--host-masks 100] [--host-noisy 4]

Inputs: blob-shaped masks (object-like), as bool masks and bit-packed as in a C3 ResultRecord, and the masks of a
seeded RSPrompterQuery ViT-B predict (random weights: noisy masks, the worst case for run-length encoding).  Device
times: CUDA events around the two kernel passes (length + scan, write) after a warm-up, and the wall clock of the
whole call (two host synchronisations, the device->host copy of the strings, slicing).  The host path is timed on a
subset of the masks and scaled to 800; it is printed as such.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, M, H, W = 8, 100, 1024, 1024


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, limit = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=limit)


def _blobs(n: int, seed: int) -> torch.Tensor:
    """n masks of 1-3 filled ellipses (radii 20-150 px) on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    yy = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1)
    xx = torch.arange(W, device="cuda", dtype=torch.float32).view(1, 1, W)
    out = torch.zeros(n, H, W, dtype=torch.bool, device="cuda")
    for _ in range(3):
        c = torch.rand(n, 2, generator=g, device="cuda") * 800 + 100
        r = torch.rand(n, 2, generator=g, device="cuda") * 130 + 20
        keep = torch.rand(n, generator=g, device="cuda") < 0.7
        cy, cx, ry, rx = (v.view(n, 1, 1) for v in (c[:, 0], c[:, 1], r[:, 0], r[:, 1]))
        e = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
        out |= (e < 1) & keep.view(n, 1, 1)
    return out


def _kernel_ms(groups, packed: bool, iters: int) -> float:
    """CUDA-event time of the length pass + offset scan + write pass (the pool is sized once, outside the window)."""
    import ctypes
    from rsprompter_b200 import _lib
    base = min(t.data_ptr() for t, _ in groups)
    rows = []
    for t, w in groups:
        n, h, ld = t.shape
        rows += [(t.data_ptr() - base + j * h * ld, h, w) for j in range(n)]
    n = len(rows)
    desc_host = torch.tensor(rows, dtype=torch.int64)
    desc = desc_host.cuda()
    offsets = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    lengths = torch.empty(n, dtype=torch.int32, device="cuda")
    lib, s = _lib._lib, torch.cuda.current_stream().cuda_stream
    dh = ctypes.c_void_p(desc_host.data_ptr())
    assert lib.rsp_mask_rle_lengths(base, int(packed), desc.data_ptr(), dh, n, offsets.data_ptr(), s) == 0
    pool = torch.empty(int(offsets[n].item()), dtype=torch.uint8, device="cuda")

    def run():
        assert lib.rsp_mask_rle_lengths(base, int(packed), desc.data_ptr(), dh, n, offsets.data_ptr(), s) == 0
        assert lib.rsp_mask_rle_write(base, int(packed), desc.data_ptr(), n, offsets.data_ptr(), pool.data_ptr(),
                                      lengths.data_ptr(), s) == 0

    for _ in range(3):
        run()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        run()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def _call_ms(fn, iters: int) -> float:
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t) / iters * 1e3


def _host_ms_per_mask(masks: torch.Tensor) -> float:
    """.cpu() of bool masks + mask_to_coco_rle per mask, as CocoMetric.process does (one core)."""
    from rsprompter_b200.results import mask_to_coco_rle
    torch.cuda.synchronize()
    t = time.perf_counter()
    host = masks.cpu().numpy()
    for m in host:
        mask_to_coco_rle(m)
    return (time.perf_counter() - t) / masks.shape[0] * 1e3


def _case(name: str, masks: list, iters: int, host_masks: int) -> dict:
    """masks: per-image CUDA bool [M, H, W]."""
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import encode_mask_results, mask_to_coco_rle
    n = sum(m.shape[0] for m in masks)
    out = encode_mask_results(masks)
    flat = [r for per_img in out for r in per_img]
    sub = torch.cat(masks)[:host_masks]
    assert [r["counts"] for r in flat[:host_masks]] == [mask_to_coco_rle(m)["counts"] for m in sub.cpu().numpy()]
    pool = sum(len(r["counts"]) for r in flat)
    bits = [_lib.pack_mask_bits(m) for m in masks]
    host_ms = _host_ms_per_mask(sub)
    res = dict(case=name, masks=n, rle_bytes=pool,
               d2h_bytes_new=pool + 4 * n + 8, d2h_bytes_bool=n * H * W, d2h_bytes_bits=n * H * W // 8,
               kernel_ms_bool=_kernel_ms([(m, W) for m in masks], False, iters),
               kernel_ms_bits=_kernel_ms([(b, W) for b in bits], True, iters),
               call_ms_bool=_call_ms(lambda: encode_mask_results(masks), iters),
               call_ms_bits=_call_ms(lambda: _lib.mask_rle([(b, W) for b in bits], packed=True), iters),
               host_ms_per_mask=host_ms, host_masks_timed=int(sub.shape[0]),
               host_ms_scaled_to_all_masks=host_ms * n)
    print(f"{name}: {n} masks, {pool / 1e6:.2f} MB of RLE | device kernels bool {res['kernel_ms_bool']:.3f} ms, "
          f"bits {res['kernel_ms_bits']:.3f} ms | whole call bool {res['call_ms_bool']:.1f} ms, bits "
          f"{res['call_ms_bits']:.1f} ms | host .cpu()+numpy RLE {host_ms:.2f} ms/mask on {res['host_masks_timed']} "
          f"masks -> {res['host_ms_scaled_to_all_masks'] / 1e3:.2f} s scaled to {n} | D2H {res['d2h_bytes_new'] / 1e6:.2f}"
          f" MB vs {res['d2h_bytes_bool'] / 1e6:.0f} MB bool / {res['d2h_bytes_bits'] / 1e6:.0f} MB bits", flush=True)
    return res


def _query_masks() -> list:
    from rsprompter_b200 import model_configs, sam_config, synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    from rsprompter_b200.registry import MODELS
    m = MODELS.build(model_configs.query_model_cfg("base", 10, prompt_shape=(M, 5)))
    arch = sam_config.VISION_ARCHS["base"]
    m.load_state_dict(synthetic.query_detector_state_dict(arch, 10, len(SELECT_LAYERS["base"]), nq=M, seed=8), strict=True)
    m = m.cuda()
    torch.manual_seed(8)
    out = m.predict(torch.randn(B, 3, H, W).cuda())
    masks = [o.pred_instances.masks.contiguous() for o in out]
    del m
    return masks


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-masks", type=int, default=100, help="blob masks timed on the host path")
    ap.add_argument("--host-noisy", type=int, default=4, help="predict masks timed on the host path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rle_bench.py needs a CUDA device (device times are not estimated on the host)")
    card = _card()
    print(f"{card['gpu']}, power limit {card['power_limit']}", flush=True)
    blobs = _blobs(B * M, seed=0)
    rows = [_case("blobs", list(blobs.view(B, M, H, W)), args.iters, args.host_masks)]
    del blobs
    rows.append(_case("query_vitb_predict", _query_masks(), args.iters, args.host_noisy))
    print(json.dumps(dict(card, cases=rows)))


if __name__ == "__main__":
    main()
