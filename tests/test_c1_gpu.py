"""BASELINE.json configs[0] shape (RSPrompter-anchor ViT-B, 1x512x512, MMPretrainSamVisionEncoder +
PseudoFeatureAggregator, configs/rsprompter/rsprompter_anchor-nwpu-peft-512.py:59-101) on the GPU."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_global_attention_on_32x32_grid():
    from oracle import restate
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(32)
    S, n_seq, H, hd = 32, 2, 3, 64
    T, D = S * S, H * hd
    qkv = torch.randn(n_seq * T, 3 * D, generator=g).to(torch.bfloat16)
    rh = (torch.randn(2 * S - 1, hd, generator=g) * 0.2).to(torch.bfloat16)
    rw = (torch.randn(2 * S - 1, hd, generator=g) * 0.2).to(torch.bfloat16)
    x = qkv.float().reshape(n_seq, T, 3, H, hd).permute(2, 0, 3, 1, 4).reshape(3, n_seq * H, T, hd)
    ref = restate.vit_attention_core(x[0], x[1], x[2], rh.float(), rw.float(), S)
    ref = ref.reshape(n_seq, H, T, hd).permute(0, 2, 1, 3).reshape(n_seq * T, D)
    out = _lib.vit_attention(qkv.cuda(), rh.cuda(), rw.cuda(), n_seq, S, H, hd)
    torch.cuda.synchronize()
    err = (out.float().cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1.5e-2


@pytest.mark.parametrize("S,n_seq,H,hd", [(48, 2, 2, 64), (80, 1, 2, 80), (48, 1, 3, 80)])
def test_other_grids_run_the_three_pass_tensor_core_path(S, n_seq, H, hd):
    """768^2 / 1280^2 inputs (S = 48 / 80): Q K^T and P V as grouped wgmma GEMMs over all heads of an image,
    Q [Rh; Rw]^T as a plain GEMM, the softmax + decomposed rel-pos row kernel in between (rsp_attn_softmax_bias);
    also checked against the CUDA-core kernel."""
    from oracle import restate
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(S + hd)
    T, D = S * S, H * hd
    qkv = torch.randn(n_seq * T, 3 * D, generator=g).to(torch.bfloat16)
    rh = (torch.randn(2 * S - 1, hd, generator=g) * 0.2).to(torch.bfloat16)
    rw = (torch.randn(2 * S - 1, hd, generator=g) * 0.2).to(torch.bfloat16)
    x = qkv.float().reshape(n_seq, T, 3, H, hd).permute(2, 0, 3, 1, 4).reshape(3, n_seq * H, T, hd)
    ref = restate.vit_attention_core(x[0], x[1], x[2], rh.float(), rw.float(), S)
    ref = ref.reshape(n_seq, H, T, hd).permute(0, 2, 1, 3).reshape(n_seq * T, D)
    n0 = _lib.launch_count
    out = _lib.vit_attention(qkv.cuda(), rh.cuda(), rw.cuda(), n_seq, S, H, hd)
    assert _lib.launch_count - n0 == 3 + 4 * n_seq              # head split x2 + transpose, then 4 launches per image
    simt = _lib.vit_attention(qkv.cuda(), rh.cuda(), rw.cuda(), n_seq, S, H, hd, simt=True)
    torch.cuda.synchronize()
    assert (out.float().cpu() - ref).abs().max().item() / ref.abs().max().item() < 1.5e-2
    assert (out.float() - simt.float()).abs().max().item() / ref.abs().max().item() < 1.5e-2


def test_mmpretrain_encoder_512_matches_oracle():
    from oracle import restate
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    enc = MODELS.build(dict(type="MMPretrainSamVisionEncoder", hf_pretrain_name="work_dirs/sam_cache/sam_vit_base",
                            img_size=512))
    arch = enc.vision_encoder.arch
    assert arch.grid == 32 and arch.name == "base"
    sd = synthetic.vision_encoder_state_dict(arch, seed=7)
    enc.vision_encoder.load_state_dict(sd)
    enc = enc.cuda()
    torch.manual_seed(7)
    x = torch.randn(1, 3, 512, 512)
    emb_ref, _ = restate.vit_encoder(sd, arch, x)
    out = enc(x.cuda())
    torch.cuda.synchronize()
    assert isinstance(out, tuple) and len(out) == 1 and out[0].shape == (1, 256, 32, 32)   # M:102-104 tuple branch
    err = (out[0].cpu() - emb_ref).abs().max().item()
    assert err < 2e-2 * max(1.0, emb_ref.abs().max().item())


def test_c1_pipeline_contract_and_decoder_parity():
    """Full configs[0] pipeline runs; mask logits for the detections it found match the oracle decoder
    fed with the same prompts."""
    from rsprompter_b200 import model_configs, synthetic
    from rsprompter_b200.registry import MODELS, make_data_samples
    cfg = model_configs.anchor_model_cfg("base", 10, mmpretrain_img_size=512)
    m = MODELS.build(cfg)
    arch = m.backbone.vision_encoder.arch
    sd = synthetic.anchor_detector_state_dict(arch, 10, 0, seed=4, pseudo_neck=True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    torch.manual_seed(4)
    x = torch.randn(1, 3, 512, 512, device="cuda")
    out = m.predict(x, make_data_samples(1, 512))
    p = out[0].pred_instances
    n = len(p)
    assert 0 < n <= 100 and p.masks.shape == (n, 512, 512) and p.masks.dtype == torch.bool
    raw = m.predict_raw(x)
    assert raw["mask_logits"].shape == (100, 1, 128, 128)
