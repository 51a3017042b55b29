"""Greedy non-maximum merging of large scenes (merge_tile_records(nms_type='greedy_nmm')) against the hard merge, and
the union RLE encode against the placed one, on seeded records.

    python profiles/nmm_merge_bench.py [--repeats 10]

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * merge: merge_tile_records over 25, 121 and 441 tiles of 100 slots (2 500, 12 100, 44 100 candidates, 10 labels,
    seeded boxes of 4 .. 175 px in 512^2 tiles at overlap 0.25), nms against greedy_nmm (IoS 0.5), the two alternated
    call by call in one process; each call ends in its host read, so a call's time is its wall time;
  * rle: for the same scenes, each slot's mask the rectangle of its box: encode_kept_masks of greedy_nmm's keepers
    alone (the placed encode) against encode_merged_masks of its groups (the union encode of the same keepers, each
    with its absorbed members), alternated.
Times are host wall clock around whole calls (each ends in a device synchronisation) after two warm-up calls; the
median of ``--repeats`` calls is reported.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import statistics
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


def _records(n_tiles, P, M, seed, batch=8):
    from rsprompter_b200 import _lib
    from rsprompter_b200.results import ResultRecord
    g = torch.Generator().manual_seed(seed)
    recs = []
    n_rec = (n_tiles + batch - 1) // batch
    scores = (torch.randperm(n_rec * batch * M, generator=g).float() + 1) / (n_rec * batch * M + 1)
    for r in range(n_rec):
        rec = ResultRecord(batch, M, (P, P), device="cuda")
        xy = torch.rand(batch, M, 2, generator=g) * (P - 8)
        wh = 4 + torch.rand(batch, M, 2, generator=g) * (P / 3)
        b = torch.cat([xy, torch.minimum(xy + wh, torch.full_like(xy, float(P)))], dim=2)
        lab = torch.randint(0, 10, (batch, M), generator=g).float()
        s = scores[r * batch * M:(r + 1) * batch * M].view(batch, M)
        rec.rows.copy_(torch.cat([b, s[..., None], lab[..., None]], dim=2))
        rec.counts.fill_(M)
        bd = b.cuda().round()                                            # each slot's mask fills its box
        yy = torch.arange(P, device="cuda").view(1, 1, P, 1)
        xx = torch.arange(P, device="cuda").view(1, 1, 1, P)
        m = ((yy >= bd[..., 1, None, None]) & (yy < bd[..., 3, None, None]) & (xx >= bd[..., 0, None, None])
             & (xx < bd[..., 2, None, None]))
        rec.mask_bits.copy_(_lib.pack_mask_bits(m.view(batch * M, P, P).contiguous()).view_as(rec.mask_bits))
        recs.append(rec)
    return recs


def _alternate(fns: dict, repeats: int) -> dict:
    """Median ms per call of each fn, the fns called in turn."""
    for fn in fns.values():
        fn(); fn()
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t) * 1e3)
    return {k: statistics.median(v) for k, v in times.items()}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args(argv)
    assert torch.cuda.is_available(), "needs a GPU"
    from rsprompter_b200.large_image import (encode_kept_masks, encode_merged_masks, merge_tile_records,
                                             slice_origins)
    card = _card()
    P, M = 512, 100
    for side in (4 * 384 + 512, 10 * 384 + 512, 20 * 384 + 512):          # 5^2, 11^2 and 21^2 tiles
        hw = (side, side)
        org = slice_origins(hw, P, 0.25)
        recs = _records(len(org), P, M, seed=len(org))
        origins = [org[i:i + 8] for i in range(0, len(org), 8)]
        kw = dict(merge_iou_thr=0.5)
        t = _alternate({"nms": lambda: merge_tile_records(recs, origins, hw, **kw),
                        "greedy_nmm": lambda: merge_tile_records(recs, origins, hw, nms_type="greedy_nmm", **kw)},
                       args.repeats)
        hard = merge_tile_records(recs, origins, hw, **kw)
        nmm = merge_tile_records(recs, origins, hw, nms_type="greedy_nmm", **kw)
        print(json.dumps(dict(what="merge", tiles=len(org), candidates=len(org) * M, kept=int(hard["scores"].numel()),
                              groups=int(nmm["scores"].numel()), members=int(nmm["members"].shape[0]),
                              nms_ms=round(t["nms"], 3), greedy_nmm_ms=round(t["greedy_nmm"], 3), **card)),
              flush=True)
        r = _alternate({"placed": lambda: encode_kept_masks(recs, origins, nmm["source"], hw),
                        "union": lambda: encode_merged_masks(recs, origins, nmm["members"], nmm["member_offsets"],
                                                             hw)},
                       max(3, args.repeats // 2))
        print(json.dumps(dict(what="rle", tiles=len(org), masks=int(nmm["scores"].numel()),
                              union_parts=int(nmm["members"].shape[0]), placed_ms=round(r["placed"], 2),
                              union_ms=round(r["union"], 2), **card)), flush=True)


if __name__ == "__main__":
    main()
