#!/usr/bin/env python
"""profiles/decoder_bench.py -- the SAM mask decoder of the C3 step (RSPrompter-query ViT-H, bs 8, 100 queries) alone.

    python profiles/decoder_bench.py [--n 800] [--hw 64] [--points 5] [--iters 20] [--warmup 3] [--multimask]

Builds the decoder call of the query head on seeded inputs: synthetic decoder / prompt-encoder weights, a random
image embedding of B = n / 100 images and random per-query mask logits, turned into the per-prompt source pair by
rsp_mask_embed_src exactly as RSPrompterQueryHead does.  Three timed passes, each on its own:
  1. `decode` end to end with CUDA events after warm-up (ms per call);
  2. every native call `decode` makes, bracketed by CUDA events on the stream, grouped into kernel families, with
     the bytes and FLOPs each family needs computed from the call's shapes -> ms, GB/s and TFLOP/s per family;
  3. torch.profiler (CUDA activity) over the same calls: device time per kernel name.
Prints one JSON object with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from rsprompter_b200 import _lib, synthetic  # noqa: E402
from rsprompter_b200.sam_config import SamDecoderArch  # noqa: E402
from rsprompter_b200.sam_decoder import SamMaskDecoderB200  # noqa: E402

NQ = 100


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clk = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clk)


def setup(n: int, side: int, points: int, seed: int = 0):
    arch = SamDecoderArch()
    dec = SamMaskDecoderB200(arch)
    dec.load_state_dict(synthetic.mask_decoder_state_dict(arch, seed=seed + 1))
    dec = dec.cuda()
    pe = synthetic.prompt_encoder_state_dict(arch, seed=seed + 2)
    C = arch.hidden_size
    me = [pe[k].float().contiguous().cuda() for k in (
        "mask_embed.conv1.weight", "mask_embed.conv1.bias", "mask_embed.layer_norm1.weight",
        "mask_embed.layer_norm1.bias", "mask_embed.conv2.weight", "mask_embed.conv2.bias",
        "mask_embed.layer_norm2.weight", "mask_embed.layer_norm2.bias")]
    me += [pe["mask_embed.conv3.weight"].reshape(C, -1).float().contiguous().cuda(),
           pe["mask_embed.conv3.bias"].float().contiguous().cuda()]
    g = torch.Generator().manual_seed(seed)
    B = max(1, n // NQ)
    hw = side * side
    emb_rows = (0.5 * torch.randn(B * hw, C, generator=g)).cuda()
    pos_rows = torch.randn(hw, C, generator=g).cuda()
    mpp = (2.0 * torch.randn(n, 4 * side, 4 * side, generator=g)).cuda()
    sparse = (0.5 * torch.randn(n, points, C, generator=g)).cuda()
    src_pair = _lib.mask_embed_src(mpp, me, emb_rows, pos_rows, min(NQ, n), (side, side))
    return dec, pos_rows, sparse, src_pair


# ------------------------------------------------------------------ bytes / FLOPs of each native call, from its shapes
def _nb(t) -> int:
    return 0 if t is None else t.numel() * t.element_size()


def _gemm_cost(a, w, *args, **kw):
    M, K = a.shape
    N = w.shape[0]
    out_b = 4 if kw.get("out_dtype", torch.bfloat16) == torch.float32 else 2
    res = kw.get("residual")
    byts = M * K * 2 + _nb(w) + M * N * out_b + (_nb(res) if res is not None and res.shape[0] <= M else 0)
    if res is not None and res.shape[0] > M:
        byts += M * N * res.element_size()
    return 2.0 * M * N * K, byts


def _upscale_cost(a, w, bias, hyper, gh, gw, *args, **kw):
    M, K = a.shape
    P, n_out = hyper.shape[0], hyper.shape[1]
    return 2.0 * M * 128 * K, M * K * 2 + P * n_out * 16 * gh * gw * 4


def _t2i_cost(q, K, V, hw, kv_block=None):
    N, Tq, C = q.shape
    rows = K.shape[0]
    return 4.0 * N * Tq * hw * C, 2 * rows * C * 2 + 2 * _nb(q)


def _i2t_cost(Q, ktok, vtok, hw, q_block=None):
    N, Tq, C = ktok.shape
    return 4.0 * N * Tq * hw * C, Q.shape[0] * C * 2 + N * hw * C * 2


def _t2i_fused_cost(q, keys, kvw, kvb, pe_kv, hw):
    N, Tq, C = q.shape
    return 2.0 * keys.shape[0] * 256 * 256 + 4.0 * N * Tq * hw * C, keys.shape[0] * 256 * 2 + 2 * _nb(q)


def _i2t_fused_cost(keys, wq, qb, pe_q, ktok, vtok, wo, ob, ln, hw):
    N, Tq, C = ktok.shape
    R = keys.shape[0]
    return 2.0 * R * 256 * 128 * 2 + 4.0 * N * Tq * hw * C, R * 256 * 2 * 2


def _family(name: str, args, kw, n_img_rows: int) -> str:
    if name == "gemm":
        a, w = args[0], args[1]
        if a.shape[0] < n_img_rows:
            return "token-side gemm"
        if kw.get("ln64_gelu") is not None:
            return "up1 gemm (LN64 + GELU)"
        if kw.get("ln") is not None:
            return "i2t out_proj gemm (+ LN4)"
        if w.shape[0] == 256:
            return "t2i k|v gemm"
        return "i2t q gemm"
    return {"gemm_upscale_masks": "up2 gemm (GELU + hyper)", "t2i_attention": "t2i attention",
            "i2t_attention": "i2t attention", "t2i_fused": "t2i fused (k|v gemm + attention)",
            "i2t_fused": "i2t fused (q gemm + attention + out_proj + LN4)"}.get(name, "token-side " + name)


COSTS = {"gemm": _gemm_cost, "gemm_upscale_masks": _upscale_cost, "t2i_attention": _t2i_cost,
         "i2t_attention": _i2t_cost, "t2i_fused": _t2i_fused_cost, "i2t_fused": _i2t_fused_cost}
WRAPPED = ("gemm", "gemm_upscale_masks", "t2i_attention", "i2t_attention", "t2i_fused", "i2t_fused", "add_cast_bf16",
           "cast_bf16", "token_self_attention")


def per_family(run, n_img_rows: int, iters: int) -> dict:
    calls = []
    orig = {k: getattr(_lib, k) for k in WRAPPED if hasattr(_lib, k)}

    def wrap(name, fn):
        def inner(*args, **kw):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = fn(*args, **kw)
            e.record()
            cost = COSTS[name](*args, **kw) if name in COSTS else (0.0, 0)
            calls.append((_family(name, args, kw, n_img_rows), s, e, cost))
            return out
        return inner

    try:
        for k, fn in orig.items():
            setattr(_lib, k, wrap(k, fn))
        for _ in range(iters):
            run()
        torch.cuda.synchronize()
    finally:
        for k, fn in orig.items():
            setattr(_lib, k, fn)
    fam = collections.defaultdict(lambda: [0.0, 0.0, 0, 0])
    for f, s, e, (fl, by) in calls:
        r = fam[f]
        r[0] += s.elapsed_time(e) / iters
        r[1] += fl / iters
        r[2] += by // iters
        r[3] += 1
    out = {}
    for f, (ms, fl, by, cnt) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        out[f] = dict(ms=round(ms, 3), calls=cnt // iters, GB=round(by / 1e9, 3),
                      GB_s=round(by / (ms * 1e-3) / 1e9, 1) if ms > 0 and by else None,
                      TFLOP_s=round(fl / (ms * 1e-3) / 1e12, 1) if ms > 0 and fl else None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=800, help="prompts (C3: 8 images x 100 queries)")
    ap.add_argument("--hw", type=int, default=64, help="side of the image-token grid")
    ap.add_argument("--points", type=int, default=5, help="sparse points per prompt (Tt = 5 + points)")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--multimask", action="store_true")
    ap.add_argument("--trace-dir", default=None, help="also write the profiler's kernel table here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decoder_bench needs a GPU")
    torch.cuda.set_device(0)
    dec, pos_rows, sparse, src_pair = setup(args.n, args.hw, args.points)
    hw = (args.hw, args.hw)

    def run():
        return dec.decode(None, pos_rows, sparse, hw, src_pair=src_pair, multimask_output=args.multimask)

    for _ in range(args.warmup):
        run()
    torch.cuda.synchronize()
    # 1. end to end
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.iters):
        run()
    e.record()
    torch.cuda.synchronize()
    decode_ms = s.elapsed_time(e) / args.iters
    # 2. per native call, grouped
    fams = per_family(run, args.n * args.hw * args.hw, args.iters)
    # 3. profiler: device time per kernel name
    from torch.profiler import ProfilerActivity, profile
    n_prof = max(3, args.iters // 4)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            run()
        torch.cuda.synchronize()
    kern = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            kern[ev.name][0] += ev.device_time_total / 1e3 / n_prof
            kern[ev.name][1] += 1
    kernels = {k[:120]: dict(ms=round(v[0], 3), launches=v[1] // n_prof)
               for k, v in sorted(kern.items(), key=lambda kv: -kv[1][0])}
    if args.trace_dir:
        os.makedirs(args.trace_dir, exist_ok=True)
        with open(os.path.join(args.trace_dir, "decoder_kernels.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=60))
    res = dict(card=_card(), n=args.n, hw=args.hw * args.hw, tt=5 + args.points, multimask=args.multimask,
               decode_ms=round(decode_ms, 3), kernel_ms=round(sum(v["ms"] for v in kernels.values()), 3),
               families=fams, kernels=kernels)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
