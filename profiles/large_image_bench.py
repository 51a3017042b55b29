"""Whole-scene inference (rsprompter_b200.large_image.predict_large_image) on seeded synthetic scenes.

    python profiles/large_image_bench.py [--sizes 4096 8192 16384] [--configs query_vith anchor_vitb] [--repeats 2]

Configs as bench.py builds them: ``query_vith`` (C3: RSPrompter-query ViT-H, 100 queries) and ``anchor_vitb``
(RSPrompter-anchor ViT-B), seeded random weights, the reference DetDataPreprocessor, CUDA graphs on, tiles of 1024^2 in
batches of 8, overlap 0.25, merge IoU 0.25.  The scene is seeded uint8 noise held on the host, so the timing includes
its one pinned copy to the device.

Per scene: tiles, tiles/s and scene seconds (host clock around the whole predict_large_image, which ends in a host
read), and the split into the three stages timed the same way in a second pass: tile inference (run_tiles, ended by a
device synchronise), the merge (merge_tile_records: candidate count, kept count) and the RLE of the kept masks plus
the copy of the strings (encode_kept_masks).  Host synchronisations per scene are counted with torch's sync debug
mode over one whole call.  The first call per config warms up the graph capture and is not timed.  Compare tiles/s
with bench.py's images/s for the same config: the difference is the cost of slicing, merging and encoding.  Needs a
GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PREPROC = dict(type="DetDataPreprocessor", mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], bgr_to_rgb=True,
               pad_size_divisor=32)
NUM_CLASSES, NQ = 10, 100


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, limit = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=limit)


def _model(config: str):
    from rsprompter_b200 import model_configs, sam_config, synthetic
    from rsprompter_b200.model_configs import SELECT_LAYERS
    from rsprompter_b200.registry import MODELS
    arch_name = "huge" if config == "query_vith" else "base"
    arch, n_sel = sam_config.VISION_ARCHS[arch_name], len(SELECT_LAYERS[arch_name])
    if config == "query_vith":
        cfg = model_configs.query_model_cfg(arch_name, NUM_CLASSES, prompt_shape=(NQ, 5))
        sd = synthetic.query_detector_state_dict(arch, NUM_CLASSES, n_sel, nq=NQ, seed=0)
    else:
        cfg = model_configs.anchor_model_cfg(arch_name, NUM_CLASSES)
        sd = synthetic.anchor_detector_state_dict(arch, NUM_CLASSES, n_sel, seed=0)
    cfg["data_preprocessor"] = dict(PREPROC)
    m = MODELS.build(cfg)
    m.load_state_dict(sd)
    return m.cuda().enable_cuda_graphs()


def _scene(size: int, seed: int) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (size, size, 3), generator=g, dtype=torch.uint8, device="cuda").cpu()


def _host_syncs(fn) -> int:
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchroniz" in str(x.message) for x in w)


def _scene_case(model, scene: torch.Tensor, repeats: int) -> dict:
    from rsprompter_b200 import large_image as li
    H, W = scene.shape[:2]
    P = model.backbone.vision_encoder.arch.image_size
    n_tiles = len(li.slice_origins((H, W), P, 0.25))
    total = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        ds = li.predict_large_image(model, scene)
        total.append(time.perf_counter() - t)
    kept = len(ds.pred_instances.masks)
    del ds
    split = dict(tiles_s=[], merge_s=[], rle_s=[])
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        records, batches = li.run_tiles(model, scene)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        merged = li.merge_tile_records(records, batches, (H, W))
        t2 = time.perf_counter()
        li.encode_kept_masks(records, batches, merged["source"], (H, W))
        t3 = time.perf_counter()
        split["tiles_s"].append(t1 - t0)
        split["merge_s"].append(t2 - t1)
        split["rle_s"].append(t3 - t2)
        candidates = int(sum(int(r.counts[:len(b)].sum()) for r, b in zip(records, batches)))
        del records, merged
    syncs = _host_syncs(lambda: li.predict_large_image(model, scene))
    best = min(total)
    res = dict(scene=[H, W], tiles=n_tiles, scene_s=best, tiles_per_s=n_tiles / best, kept=kept,
               candidates=candidates, slots=n_tiles * li._slots(model),
               tile_inference_s=min(split["tiles_s"]), merge_s=min(split["merge_s"]), rle_and_copy_s=min(split["rle_s"]),
               host_syncs_per_scene=syncs, scene_s_all=total)
    print(f"  {H}x{W}: {n_tiles} tiles, {res['scene_s']:.2f} s/scene, {res['tiles_per_s']:.1f} tiles/s | tiles "
          f"{res['tile_inference_s']:.2f} s, merge {res['merge_s'] * 1e3:.1f} ms ({candidates} candidates of "
          f"{res['slots']} slots, {kept} kept), RLE + copy {res['rle_and_copy_s'] * 1e3:.1f} ms | {syncs} host syncs",
          flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 8192, 16384])
    ap.add_argument("--configs", nargs="+", default=["query_vith", "anchor_vitb"], choices=["query_vith", "anchor_vitb"])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("large_image_bench.py needs a CUDA device (device times are not estimated on the host)")
    from rsprompter_b200 import large_image as li
    card = _card()
    print(f"{card['gpu']}, power limit {card['power_limit']}", flush=True)
    rows = []
    for config in args.configs:
        model = _model(config)
        print(config, flush=True)
        li.predict_large_image(model, _scene(2048, 0))        # graph capture + warm-up, not timed
        for size in args.sizes:
            rows.append(dict(config=config, **_scene_case(model, _scene(size, size), args.repeats)))
        del model
        torch.cuda.empty_cache()
    text = json.dumps(dict(card, cases=rows))
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
