"""The north-star model at full depth: SAM ViT-H (32 layers, D 1280, 16 heads of 80) 1024^2 on the GPU against the
fp32 CPU restatement, EVERY hidden state, with the per-layer error growth written to gpurun_out/ (SURVEY 8 row a1)."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dump(name: str, obj) -> None:
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", name), "w") as f:
            json.dump(obj, f, indent=1)
    except OSError:
        pass


def test_vith_32_layer_encoder_matches_oracle():
    from oracle import restate
    from rsprompter_b200 import synthetic
    from rsprompter_b200.sam_config import VISION_ARCHS
    from rsprompter_b200.sam_encoder import SamVisionEncoderB200
    arch = VISION_ARCHS["huge"]
    assert arch.num_layers == 32 and arch.hidden_size == 1280 and arch.head_dim == 80
    sd = synthetic.vision_encoder_state_dict(arch, seed=5)
    torch.manual_seed(5)
    x = torch.randn(1, 3, 1024, 1024)
    with torch.no_grad():
        emb_ref, hid_ref = restate.vit_encoder(sd, arch, x)
    enc = SamVisionEncoderB200(arch)
    enc.load_state_dict(sd)
    enc = enc.cuda()
    emb, hid, _ = enc.encode(x.cuda())
    torch.cuda.synchronize()
    assert len(hid) == 33 and tuple(hid[0].shape) == (1, 64, 64, 1280)
    rows = []
    for i, (h, r) in enumerate(zip(hid, hid_ref)):
        d = (h.cpu() - r).abs()
        rows.append(dict(hidden_state=i, max_abs_err=d.max().item(), mean_abs_err=d.mean().item(),
                         max_abs_ref=r.abs().max().item(), rms_ref=r.pow(2).mean().sqrt().item()))
    e = (emb.cpu() - emb_ref).abs()
    summary = dict(layers=rows, embedding=dict(max_abs_err=e.max().item(), mean_abs_err=e.mean().item(),
                                               max_abs_ref=emb_ref.abs().max().item()))
    _dump("parity_vith_encoder.json", summary)
    print("ViT-H per-layer max|err| / max|ref|:",
          " ".join(f"{r['max_abs_err']:.3g}/{r['max_abs_ref']:.3g}" for r in rows[::4]), "| embedding",
          f"{summary['embedding']['max_abs_err']:.3g}/{summary['embedding']['max_abs_ref']:.3g}")
    # tolerance: bf16 operands with fp32 accumulation and an fp32 residual stream: 2e-2 relative to the tensor's range
    # for the hidden states (their range grows with depth), 2e-2 ABSOLUTE x range for the LayerNorm-ed embedding
    for r in rows:
        assert r["max_abs_err"] <= 2e-2 * max(1.0, r["max_abs_ref"]), r
    assert summary["embedding"]["max_abs_err"] <= 2e-2 * max(1.0, summary["embedding"]["max_abs_ref"])


def test_lora_checkpoint_on_gpu_matches_unmerged_oracle():
    """SURVEY 8(f3): a peft-LoRA checkpoint (M:785-797 key layout) loaded into the H100 encoder (adapter folded into
    qkv.weight at load) against the oracle that keeps the adapter branch separate: y = Wx + b + (alpha/r) B(A x)."""
    from oracle import restate
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import SamVisionArch
    r, alpha = 16, 32
    enc = MODELS.build(dict(type="MMPretrainSamVisionEncoder", hf_pretrain_name="work_dirs/sam_cache/sam_vit_base",
                            img_size=512, peft_config=dict(peft_type="LORA", r=r, target_modules=["qkv"],
                                                           lora_alpha=alpha, lora_dropout=0.05, bias="none")))
    arch = enc.vision_encoder.arch
    base = synthetic.vision_encoder_state_dict(arch, seed=4)
    g = torch.Generator().manual_seed(5)
    ck, osd = {}, dict(base)
    for k, v in base.items():
        if k.endswith("attn.qkv.weight"):
            stem = "vision_encoder.base_model.model." + k[:-len(".weight")]
            A = torch.randn(r, v.shape[1], generator=g) * 0.05
            B = torch.randn(v.shape[0], r, generator=g) * 0.05
            ck[stem + ".base_layer.weight"] = v
            ck[stem + ".lora_A.default.weight"], ck[stem + ".lora_B.default.weight"] = A, B
            p = k[:-len("weight")]
            osd[p + "lora_A"], osd[p + "lora_B"], osd[p + "lora_scale"] = A, B, torch.tensor(alpha / r)
        elif k.endswith("attn.qkv.bias"):
            ck["vision_encoder.base_model.model." + k[:-len(".bias")] + ".base_layer.bias"] = v
        else:
            ck["vision_encoder.base_model.model." + k] = v
    enc.load_state_dict(ck, strict=True)
    enc = enc.cuda()
    torch.manual_seed(6)
    x = torch.randn(1, 3, 512, 512)
    with torch.no_grad():
        emb_ref, _ = restate.vit_encoder(osd, arch, x)
        emb_base, _ = restate.vit_encoder(base, arch, x)
    out = enc(x.cuda())[0]
    torch.cuda.synchronize()
    err = (out.cpu() - emb_ref).abs().max().item()
    moved = (emb_base - emb_ref).abs().max().item()
    assert moved > 10 * err, f"the adapter must matter for this test to mean anything (moved {moved}, err {err})"
    assert err < 2e-2 * max(1.0, emb_ref.abs().max().item())
