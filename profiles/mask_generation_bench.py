"""Segment-everything (rsprompter_b200.mask_generation.generate_masks) on seeded synthetic weights and images.

    python profiles/mask_generation_bench.py [--archs base huge] [--repeats 3] [--out result.json]

Workloads: ViT-B and ViT-H, images of 1024 x 1024 and 600 x 800 (seeded smooth uint8 noise), the default 32 x 32 grid
in calls of 64 prompts, with HF's default thresholds and with every threshold 0 (filters off: every one of the 3072
candidates reaches the NMS, the worst case, and what random weights give).  Per workload:

  * call_ms: one whole generate_masks(output_rle_mask=True) call, host clock around it (it ends in host reads), best
    of the repeats;
  * the split, each stage ended by a device synchronise: encoder, decoder + stats + filter (every call of the grid),
    NMS (with its one host read), paste + RLE (with its two host reads); stats_ms is rsp_sam_mask_stats alone over the
    same calls' logits, timed with CUDA events, and decoder_ms = that stage minus stats_ms;
  * stats kernel rates: output pixels evaluated per second (3072 x H x W per image) and the logits it reads once, over
    its time (the 16 taps of each pixel come from L1 / L2, not counted);
  * hf_post_ms: the same post-processing done HF's way on the GPU on the same decoder outputs
    (SamImageProcessor.post_process_masks(binarize=False) + filter_masks per call, post_process_for_mask_generation
    once), alternated in this process with ours_post_ms (rsp_sam_mask_stats per call + NMS + paste + RLE), best of
    the repeats each; "not measured" when transformers does not import.

The card's name and power limit are printed with the numbers.  Needs a GPU: without one it fails."""
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

GRID, PPB = 32, 64
THRESHOLDS = {"hf_default": dict(pred_iou_thresh=0.88, stability_score_thresh=0.95),
              "zero": dict(pred_iou_thresh=0.0, stability_score_thresh=0.0)}


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


def _image(hw, seed):
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, 8, 8, generator=g) * 255, hw, mode="bilinear", align_corners=False)[0]
    return (base + 20 * torch.rand(3, *hw, generator=g)).clamp(0, 255).to(torch.uint8).cuda()


def _sync_ms(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


def _stats_pass(cand, p):
    """rsp_sam_mask_stats over every call's logits, as _candidates runs it; fills cand's keep / boxes / stability."""
    from rsprompter_b200 import _lib
    n_out = cand["n_out"]
    rows = PPB * n_out
    total = cand["logits"].shape[0]
    geom = ((1024, 1024), cand["reshaped"][0], cand["sizes"][0])
    iou, keep, boxes, stab = (cand[k].view(total, *cand[k].shape[2:]) for k in ("iou", "keep", "boxes", "stability"))
    for r0 in range(0, total, rows):
        r1 = min(total, r0 + rows)
        _, bx, st, kp = _lib.sam_mask_stats(cand["logits"][r0:r1], geom, 0.0, 1.0, iou[r0:r1], p["pred_iou_thresh"],
                                            p["stability_score_thresh"])
        boxes[r0:r1].copy_(bx)
        stab[r0:r1].copy_(st)
        keep[r0:r1].copy_(kp)


def _stats_kernel_ms(cand, p, reps=5):
    _stats_pass(cand, p)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        _stats_pass(cand, p)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _hf_post(proc, cand, p, nms_thr=0.7):
    hw, rs = cand["sizes"][0], cand["reshaped"][0]
    H, W = hw
    low = cand["logits"].view(-1, 3, *cand["logits"].shape[-2:])
    iou = cand["iou"].view(-1, 3)
    masks_all, scores_all, boxes_all = [], [], []
    for q0 in range(0, low.shape[0], PPB):
        masks = proc.post_process_masks([low[q0:q0 + PPB]], [hw], [rs], mask_threshold=0.0, binarize=False)[0]
        rle, scores, boxes = proc.filter_masks(masks, iou[q0:q0 + PPB], hw, [0, 0, W, H], p["pred_iou_thresh"],
                                               p["stability_score_thresh"], 0.0, 1.0)
        masks_all.extend(rle)
        scores_all.append(scores)
        boxes_all.append(boxes)
    out = proc.post_process_for_mask_generation(masks_all, torch.cat(scores_all), torch.cat(boxes_all), nms_thr)
    return len(out[0])


def _nms(cand):
    from rsprompter_b200 import mask_generation as mg
    return mg._nms(cand["iou"], cand["keep"], cand["boxes"], 0.7)


def _paste_rle(cand, idx, counts, idx_host):
    """The kept masks pasted as bits, then their COCO RLE, as generate_masks(output_rle_mask=True) does."""
    from rsprompter_b200 import mask_generation as mg
    out = mg._outputs(cand, idx, counts, idx_host, 0.0, 1024)
    mg._add_rle(out)
    return out


def _ours_post(cand, p):
    _stats_pass(cand, p)
    idx, counts, idx_host = _nms(cand)
    _paste_rle(cand, idx, counts, idx_host)
    return counts[0]


def _case(model, arch_name, hw, tname, repeats, proc) -> dict:
    from rsprompter_b200 import mask_generation as mg
    sm = model.sam_model
    img = _image(hw, hw[0] + hw[1])
    p = dict(points_per_side=GRID, points_per_batch=PPB, stability_score_offset=1.0, mask_threshold=0.0,
             **THRESHOLDS[tname])
    kw = dict(points_per_side=GRID, points_per_batch=PPB, output_rle_mask=True, **THRESHOLDS[tname])
    mg.generate_masks(model, img, **kw)                                          # warm-up
    call = min(_sync_ms(lambda: mg.generate_masks(model, img, **kw))[1] for _ in range(repeats))
    split = dict(encoder_ms=[], decode_stats_filter_ms=[], nms_ms=[], paste_rle_ms=[])
    for _ in range(repeats):
        (pix, sizes, reshaped), _ = _sync_ms(lambda: mg._inputs(sm, img, None, None, None, img.device))
        emb, t_enc = _sync_ms(lambda: sm._encode(pix))
        cand, t_dec = _sync_ms(lambda: mg._candidates(sm, emb, sizes, reshaped, p))
        (idx, counts, idx_host), t_nms = _sync_ms(lambda: _nms(cand))
        out, t_out = _sync_ms(lambda: _paste_rle(cand, idx, counts, idx_host))
        for k, v in zip(split, (t_enc, t_dec, t_nms, t_out)):
            split[k].append(v)
    n_cand = cand["logits"].shape[0]
    stats_ms = _stats_kernel_ms(cand, p)
    H, W = hw
    res = dict(arch=arch_name, image=[H, W], thresholds=tname, grid=GRID, points_per_batch=PPB, call_ms=call,
               **{k: min(v) for k, v in split.items()}, stats_ms=stats_ms,
               candidates=n_cand, after_filter=int(cand["keep"].sum()), kept=int(counts[0]),
               stats_gpix_per_s=n_cand * H * W / stats_ms / 1e6,
               stats_logit_gb_per_s=cand["logits"].numel() * 4 / stats_ms / 1e6)
    res["decoder_ms"] = res["decode_stats_filter_ms"] - stats_ms
    if proc is None:
        res["hf_post_ms"] = res["ours_post_ms"] = "not measured"
    else:
        hf, ours = [], []
        for _ in range(repeats):
            n_hf, t = _sync_ms(lambda: _hf_post(proc, cand, p))
            hf.append(t)
            n_ours, t = _sync_ms(lambda: _ours_post(cand, p))
            ours.append(t)
        res.update(hf_post_ms=min(hf), ours_post_ms=min(ours), hf_kept=n_hf, ours_kept=n_ours)
    print(f"  {arch_name} {H}x{W} {tname}: call {call:.1f} ms | encoder {res['encoder_ms']:.1f}, decoder "
          f"{res['decoder_ms']:.1f}, stats {stats_ms:.2f} ({res['stats_gpix_per_s']:.1f} Gpix/s), NMS "
          f"{res['nms_ms']:.2f}, paste + RLE {res['paste_rle_ms']:.2f} ms | {n_cand} candidates, "
          f"{res['after_filter']} filtered in, {res['kept']} kept | post-processing HF {res['hf_post_ms']} ms vs "
          f"ours {res['ours_post_ms']} ms", flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--archs", nargs="+", default=["base", "huge"], choices=["base", "large", "huge"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mask_generation_bench.py needs a CUDA device (device times are not estimated on the host)")
    try:
        from transformers import SamImageProcessor
        proc = SamImageProcessor()
    except Exception as e:                      # the HF comparison is optional; ours is timed regardless
        print(f"transformers unavailable ({e}): HF post-processing not measured", flush=True)
        proc = None
    card = _card()
    print(f"{card['gpu']}, power limit {card['power_limit']}", flush=True)
    rows = []
    with torch.no_grad():
        for arch_name in args.archs:
            model = _model(arch_name)
            for hw in ((1024, 1024), (600, 800)):
                for tname in THRESHOLDS:
                    rows.append(_case(model, arch_name, hw, tname, args.repeats, proc))
            del model
            torch.cuda.empty_cache()
    text = json.dumps(dict(card, cases=rows))
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
