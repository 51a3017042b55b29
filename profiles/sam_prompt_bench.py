"""Point-prompted SAM decoding on cached image embeddings, and the fused three-output upscale against the three
single-output launches it replaces.

    python profiles/sam_prompt_bench.py [--repeats 20] [--archs base huge]

For each ViT arch (synthetic seeded weights), one 1024^2 image is encoded once (get_image_embeddings), then
RSSamModel(image_embeddings=..., one positive point per prompt, multimask_output=True) is timed at point_batch 1, 64 and
256.  The up2 GEMM of the same shapes is timed both ways, the two alternated in one process, with their outputs
compared (torch.equal).  Device times are CUDA events over ``--repeats`` calls after two warm-up calls.  Prints one JSON
line per measurement with the card's name and power limit read in the same run.  Needs a GPU: without one it fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    name, power = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return dict(gpu=name, power_limit=power)


def _time(fn, repeats: int) -> float:
    """ms per call, CUDA events."""
    fn(); fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeats


def _model(arch_name: str):
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch
    arch, darch = VISION_ARCHS[arch_name], SamDecoderArch()
    sd = {"shared_image_embedding.positional_embedding":
          synthetic.positional_embedding_state_dict(arch, 3)["positional_embedding"]}
    sd.update({"vision_encoder." + k: v for k, v in synthetic.vision_encoder_state_dict(arch, 0).items()})
    sd.update({"mask_decoder." + k: v for k, v in synthetic.mask_decoder_state_dict(darch, 1).items()})
    sd.update({"prompt_encoder." + k: v for k, v in synthetic.prompt_encoder_state_dict(darch, 2).items()})
    m = MODELS.build(dict(type="RSSamModel", hf_pretrain_name=f"facebook/sam-vit-{arch_name}"))
    m.sam_model.load_state_dict(sd, strict=True)
    return m.cuda()


def main() -> None:
    from rsprompter_b200 import _lib
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--archs", nargs="+", default=["base", "huge"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sam_prompt_bench needs a GPU"
    card = _card()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 3, 1024, 1024, generator=g).cuda()
    for arch in args.archs:
        model = _model(arch)
        enc_ms = _time(lambda: model.get_image_embeddings(x), 3)
        emb = model.get_image_embeddings(x)
        print(json.dumps(dict(kind="encode", arch=arch, ms=round(enc_ms, 3), **card)), flush=True)
        for pb in (1, 64, 256):
            pts = (torch.rand(1, pb, 1, 2, generator=g) * 1023).cuda()
            lab = torch.ones(1, pb, 1, dtype=torch.int32).cuda()
            ms = _time(lambda: model(image_embeddings=emb, input_points=pts, input_labels=lab, multimask_output=True),
                       args.repeats)
            print(json.dumps(dict(kind="decode_points", arch=arch, point_batch=pb, multimask=True, ms=round(ms, 3),
                                  prompts_per_s=round(pb * 1000.0 / ms, 1), **card)), flush=True)
        del model
        torch.cuda.empty_cache()
    # the up2 GEMM: one fused three-output launch against three single-output launches + the stack of HF's layout
    for pb in (1, 64, 256):
        up1 = torch.randn(pb * 4 * 64 * 64, 64, generator=g).to(torch.bfloat16).cuda()
        w = (torch.randn(128, 64, generator=g) * 0.2).to(torch.bfloat16).cuda()
        b = (torch.randn(128, generator=g) * 0.1).cuda()
        hyper = torch.randn(pb, 3, 32, generator=g).cuda()
        hs = [hyper[:, o].contiguous() for o in range(3)]
        fused = lambda: _lib.gemm_upscale_masks(up1, w, b, hyper, 64, 64)  # noqa: E731
        single = lambda: torch.stack([_lib.gemm_upscale_mask(up1, w, b, h, 64, 64) for h in hs], dim=1)  # noqa: E731
        equal = bool(torch.equal(fused(), single()))
        tf, ts = [], []
        for _ in range(3):                      # alternated
            tf.append(_time(fused, args.repeats))
            ts.append(_time(single, args.repeats))
        print(json.dumps(dict(kind="upscale_up2", prompts=pb, fused_ms=round(min(tf), 4), single_x3_ms=round(min(ts), 4),
                              fused_ms_all=[round(t, 4) for t in tf], single_x3_ms_all=[round(t, 4) for t in ts],
                              outputs_equal=equal, **card)), flush=True)


if __name__ == "__main__":
    main()
