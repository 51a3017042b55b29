"""Host-side contract of the registry modules, checked without a GPU: construction through
MODELS.build, reference parameter names (state dicts load strictly), C-ABI symbol table."""
import ctypes
import os
import re

import pytest
import torch

import rsprompter_b200 as rb
from rsprompter_b200 import _lib, synthetic
from rsprompter_b200.registry import MODELS
from rsprompter_b200.sam_config import SamDecoderArch, SamVisionArch, VISION_ARCHS, parse_arch_name

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_binding_and_library_export_the_same_abi_3_symbols():
    hdr = open(os.path.join(ROOT, "include", "rsp_b200.h")).read()
    declared = set(re.findall(r"\b(rsp_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.declared_symbols())
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    for name in declared:
        assert hasattr(lib, name), f"{name} missing from librsp_b200.so"
    assert lib.rsp_abi_version() == 3


def test_arch_name_parsing():
    assert parse_arch_name("facebook/sam-vit-huge") == "huge"
    assert parse_arch_name("work_dirs/sam_cache/sam_vit_base") == "base"
    assert parse_arch_name("facebook/sam-vit-large") == "large"
    with pytest.raises(ValueError):
        parse_arch_name("resnet50")


@pytest.mark.parametrize("name", ["base", "huge"])
def test_encoder_state_dict_names_match_reference(name):
    arch = VISION_ARCHS[name]
    enc = MODELS.build(dict(type="RSSamVisionEncoder", hf_pretrain_name=f"facebook/sam-vit-{name}",
                            extra_config=dict(output_hidden_states=True)))
    sd = synthetic.vision_encoder_state_dict(arch, seed=0)
    assert set(enc.vision_encoder.state_dict()) == set(sd)
    enc.vision_encoder.load_state_dict(sd, strict=True)
    assert enc.vision_encoder.arch.output_hidden_states
    hd = arch.head_dim
    assert enc.vision_encoder.layers[0].attn.rel_pos_h.shape == (27, hd)
    g = arch.global_attn_indexes[0]
    assert enc.vision_encoder.layers[g].attn.rel_pos_h.shape == (127, hd)


def test_decoder_and_prompt_modules_load_reference_names():
    dec = MODELS.build(dict(type="RSSamMaskDecoder", hf_pretrain_name="facebook/sam-vit-base"))
    sd = synthetic.mask_decoder_state_dict(SamDecoderArch(), seed=1)
    assert set(dec.mask_decoder.state_dict()) == set(sd)
    dec.mask_decoder.load_state_dict(sd, strict=True)
    pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base"))
    pe.prompt_encoder.load_state_dict(synthetic.prompt_encoder_state_dict(SamDecoderArch(), seed=2), strict=True)
    assert pe.prompt_encoder.no_mask_embed.weight.shape == (1, 256)
    pos = MODELS.build(dict(type="RSSamPositionalEmbedding", hf_pretrain_name="facebook/sam-vit-base"))
    assert pos.shared_image_embedding.positional_embedding.shape == (2, 128)


def test_no_cpu_fallback():
    arch = SamVisionArch("tiny", 128, 1, 2, 256, (0,), image_size=1024)
    from rsprompter_b200.sam_encoder import SamVisionEncoderB200
    enc = SamVisionEncoderB200(arch)
    enc.load_state_dict(synthetic.vision_encoder_state_dict(arch, seed=0))
    with pytest.raises(_lib.RspError):
        enc.encode(torch.zeros(1, 3, 1024, 1024))


def test_window_map_matches_window_partition():
    from oracle import restate
    from rsprompter_b200.sam_encoder import window_maps
    B, g, ws = 2, 64, 14
    wmap, n_win = window_maps(B, g, ws, torch.device("cpu"))
    tok = torch.arange(B * g * g, dtype=torch.float32).reshape(B, g, g, 1) + 1
    ref, _ = restate.window_partition(tok, ws)
    ref = ref.reshape(-1).long() - 1          # padding (0) -> -1
    assert n_win == 25 and torch.equal(wmap.long(), ref)


def test_metas_crop_geometry_follows_reference_formulas():
    """detectors._SamDetectorBase._metas: fast path only for untouched images; crop = int(ori * scale_factor)
    clipped to the batch shape (M:1771-1773, M:681-685)."""
    import torch
    from rsprompter_b200.detectors import _SamDetectorBase
    from rsprompter_b200.registry import make_data_samples
    x = torch.empty(3, 3, 1024, 1024)
    ds = make_data_samples(3, (1024, 1024))
    ds[1].set_metainfo(dict(ori_shape=(512, 512), img_shape=(1024, 1024), scale_factor=(2.0, 2.0)))
    ds[2].set_metainfo(dict(ori_shape=(600, 800), img_shape=(768, 1024), scale_factor=(1.28, 1.28)))
    hw, metas = _SamDetectorBase._metas(ds, x)
    assert hw == (1024, 1024) and metas[0] is None
    assert metas[1] == dict(ori_hw=(512, 512), crop_hw=(1024, 1024), scale_factor=(2.0, 2.0))
    assert metas[2]["crop_hw"] == (int(600 * 1.28), int(800 * 1.28)) == (768, 1024) and metas[2]["ori_hw"] == (600, 800)


def test_cuda_graph_cache_is_dropped_when_weights_change():
    """Captured graphs reference the prepared (bf16, re-laid-out) weights: loading a state dict must invalidate them."""
    from rsprompter_b200 import model_configs, sam_config, synthetic
    from rsprompter_b200.registry import MODELS
    m = MODELS.build(model_configs.anchor_model_cfg("base", 3, mmpretrain_img_size=512))
    m.enable_cuda_graphs()
    m._graphs[("fake",)] = object()
    arch = m.backbone.vision_encoder.arch
    m.load_state_dict(synthetic.anchor_detector_state_dict(arch, 3, 0, seed=1, pseudo_neck=True))
    assert m._graphs == {}
    m._graphs[("fake",)] = object()
    m.float()
    assert m._graphs == {}
    assert m.enable_cuda_graphs(False)._graphs is None


def test_det_data_preprocessor_matches_documented_semantics():
    """BGR->RGB, float, (x - mean) / std, pad bottom/right to the divisor, metainfo (data_preprocessor.py:110-149 over
    mmengine ImgDataPreprocessor.forward / stack_batch, restated with numpy)."""
    import numpy as np
    import torch
    from rsprompter_b200.registry import MODELS, make_data_samples
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    pp = MODELS.build(dict(type="DetDataPreprocessor", mean=mean, std=std, bgr_to_rgb=True, pad_mask=True,
                           pad_size_divisor=32, batch_augments=[dict(type="BatchFixedSizePad", size=(64, 64))]))
    assert list(pp.state_dict()) == []                       # nothing a reference checkpoint would not have
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (3, 50, 70), generator=g, dtype=torch.uint8),
            torch.randint(0, 256, (3, 64, 33), generator=g, dtype=torch.uint8)]
    ds = make_data_samples(2, (64, 64))
    out = pp(dict(inputs=imgs, data_samples=ds))
    m, s = np.array(mean, np.float32).reshape(3, 1, 1), np.array(std, np.float32).reshape(3, 1, 1)
    ref = np.zeros((2, 3, 64, 96), np.float32)
    for i, t in enumerate(imgs):
        a = (t.numpy()[::-1].astype(np.float32) - m) / s
        ref[i, :, :a.shape[1], :a.shape[2]] = a
    assert out["inputs"].shape == (2, 3, 64, 96) and np.abs(out["inputs"].numpy() - ref).max() < 1e-6
    assert [d.metainfo["pad_shape"] for d in out["data_samples"]] == [(64, 96), (64, 64)]
    assert all(d.metainfo["batch_input_shape"] == (64, 96) for d in out["data_samples"])
    batched = pp(dict(inputs=torch.stack([imgs[0], imgs[0]]), data_samples=None))      # default_collate form
    assert batched["inputs"].shape == (2, 3, 64, 96) and torch.equal(batched["inputs"][0], out["inputs"][0])


def test_peft_lora_checkpoint_is_merged_on_load():
    """A state dict with the reference's peft key layout (M:785-797) loads into the plain encoder with
    W_qkv += (lora_alpha / r) * B @ A."""
    import torch
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    enc = MODELS.build(dict(type="MMPretrainSamVisionEncoder", hf_pretrain_name="work_dirs/sam_cache/sam_vit_base",
                            img_size=512, peft_config=dict(peft_type="LORA", r=16, target_modules=["qkv"], lora_alpha=32,
                                                           lora_dropout=0.05, bias="none")))
    arch = enc.vision_encoder.arch
    base = synthetic.vision_encoder_state_dict(arch, seed=4)
    g = torch.Generator().manual_seed(5)
    ck = {}
    for k, v in base.items():
        if k.endswith("attn.qkv.weight"):
            stem = "vision_encoder.base_model.model." + k[:-len(".weight")]
            A, B = torch.randn(16, v.shape[1], generator=g) * 0.02, torch.randn(v.shape[0], 16, generator=g) * 0.02
            ck[stem + ".base_layer.weight"] = v
            ck[stem + ".lora_A.default.weight"], ck[stem + ".lora_B.default.weight"] = A, B
            base[k] = v + 2.0 * (B @ A)
        elif k.endswith("attn.qkv.bias"):
            ck["vision_encoder.base_model.model." + k[:-len(".bias")] + ".base_layer.bias"] = v
        else:
            ck["vision_encoder.base_model.model." + k] = v
    enc.load_state_dict(ck, strict=True)
    got = enc.vision_encoder.state_dict()
    assert set(got) == set(base)
    for k in base:
        assert torch.allclose(got[k], base[k], rtol=1e-6, atol=1e-7), k


def test_mmpretrain_named_checkpoint_loads_through_load_state_dict():
    """Keys as the reference's MMPretrainSamVisionEncoder saves them (mmpretrain ViTSAM names) load without a helper."""
    import re
    import torch
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    enc = MODELS.build(dict(type="MMPretrainSamVisionEncoder", hf_pretrain_name="work_dirs/sam_cache/sam_vit_base", img_size=512))
    base = synthetic.vision_encoder_state_dict(enc.vision_encoder.arch, seed=6)
    back = [(r"^neck\.conv1\.", "channel_reduction.0."), (r"^neck\.layer_norm1\.", "channel_reduction.1."),
            (r"^neck\.conv2\.", "channel_reduction.2."), (r"^neck\.layer_norm2\.", "channel_reduction.3."),
            (r"\.layer_norm1\.", ".ln1."), (r"\.layer_norm2\.", ".ln2."), (r"\.mlp\.lin1\.", ".ffn.layers.0.0."),
            (r"\.mlp\.lin2\.", ".ffn.layers.1.")]
    ck = {}
    for k, v in base.items():
        for pat, rep in back:
            k = re.sub(pat, rep, k)
        ck["vision_encoder." + k] = v
    assert any(".ln1." in k for k in ck) and any("channel_reduction.3." in k for k in ck)
    enc.load_state_dict(ck, strict=True)
    got = enc.vision_encoder.state_dict()
    assert all(torch.equal(got[k], base[k]) for k in base)


@pytest.mark.parametrize("fmt", ["bin", "safetensors"])
def test_init_cfg_pretrained_picks_submodule_by_prefix(tmp_path, fmt):
    """One HF-style SamModel checkpoint file (prefixes vision_encoder. / mask_decoder. / prompt_encoder. /
    shared_image_embedding.) initialises each registry module through init_cfg, as the reference configs do
    (_base_/rsprompter_anchor.py:61-70,135-138; revise_keys at M:783, M:909)."""
    import torch
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS
    dec = synthetic.mask_decoder_state_dict(seed=31)
    pe = synthetic.prompt_encoder_state_dict(seed=32)
    pos = synthetic.positional_embedding_state_dict(VISION_ARCHS["base"], 33)
    ck = {"mask_decoder." + k: v for k, v in dec.items()}
    ck.update({"prompt_encoder." + k: v for k, v in pe.items()})
    ck.update({"shared_image_embedding." + k: v for k, v in pos.items()})
    ck["vision_encoder.pos_embed"] = torch.zeros(1, 2, 2, 4)          # ignored by the non-encoder modules
    path = str(tmp_path / ("model." + fmt))
    if fmt == "bin":
        torch.save(ck, path)
    else:
        from safetensors.torch import save_file
        save_file({k: v.contiguous() for k, v in ck.items()}, path)
    init = dict(type="Pretrained", checkpoint=path)
    d = MODELS.build(dict(type="RSSamMaskDecoder", hf_pretrain_name="facebook/sam-vit-base", init_cfg=init))
    e = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base", init_cfg=init))
    s = MODELS.build(dict(type="RSSamPositionalEmbedding", hf_pretrain_name="facebook/sam-vit-base", init_cfg=init))
    got = d.mask_decoder.state_dict()
    assert all(torch.equal(got[k], v) for k, v in dec.items())
    assert torch.equal(e.prompt_encoder.mask_embed.conv3.weight, pe["mask_embed.conv3.weight"])
    assert torch.equal(s.shared_image_embedding.positional_embedding, pos["positional_embedding"])


def test_rssammodel_state_dict_names_match_hf_sammodel():
    """RSSamModel.sam_model (SURVEY 8(f4), M:718-741) carries HF SamModel's parameter names and shapes (ViT-B)."""
    import torch
    from transformers import SamConfig, SamModel
    with torch.device("meta"):
        hf = SamModel(SamConfig())
    m = MODELS.build(dict(type="RSSamModel", hf_pretrain_name="facebook/sam-vit-base"))
    ours = {k: tuple(v.shape) for k, v in m.sam_model.state_dict().items()}
    ref = {k: tuple(v.shape) for k, v in hf.state_dict().items()}
    assert ours == ref


def test_oracle_embed_boxes_matches_hf_prompt_encoder():
    import torch
    from transformers import SamConfig
    from transformers.models.sam.modeling_sam import SamPromptEncoder
    from oracle import restate
    torch.manual_seed(0)
    pe = SamPromptEncoder(SamConfig()).eval()
    boxes = torch.rand(2, 3, 4) * 1000
    with torch.no_grad():
        ref = pe._embed_boxes(boxes.clone())
        got = restate.embed_boxes(pe.shared_embedding.positional_embedding, pe.point_embed[2].weight,
                                  pe.point_embed[3].weight, boxes, 1024)
    assert torch.allclose(got, ref, atol=1e-5)


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype in include/rsp_b200.h against the ctypes table of _lib: same arity, and every parameter of the
    same class (pointer / integer / float).  A mismatch here would only show up as garbage arguments on a GPU."""
    hdr = open(os.path.join(ROOT, "include", "rsp_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    protos = re.findall(r"\b(?:int|const char\s*\*)\s+(rsp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == len(set(n for n, _ in protos)) == len(_lib.declared_symbols())

    def klass(param: str) -> str:
        param = param.strip()
        if "*" in param:
            return "ptr"
        base = param.rsplit(" ", 1)[0].replace("const", "").strip()
        return {"int": "int", "float": "float", "long long": "int", "int64_t": "int", "int32_t": "int", "uint8_t": "int",
                "size_t": "int"}[base]

    ctype_class = {ctypes.c_void_p: "ptr", ctypes.c_char_p: "ptr", ctypes.c_int: "int", ctypes.c_longlong: "int",
                   ctypes.c_float: "float", ctypes.c_size_t: "int"}
    for name, params in protos:
        params = [p for p in params.split(",") if p.strip() and p.strip() != "void"]
        argtypes, _ = _lib._SIGNATURES[name]
        assert len(argtypes) == len(params), f"{name}: header has {len(params)} parameters, ctypes {len(argtypes)}"
        for k, (p, t) in enumerate(zip(params, argtypes)):
            assert klass(p) == ctype_class[t], f"{name}: parameter {k} ({p.strip()}) bound as {t.__name__}"


def test_detector_meta_helpers():
    """_metas: None for images at the batch shape with scale 1 (fast batched post-process), otherwise the crop of the
    resized image (M:1771-1773: int(ori * scale), capped at the batch shape) and the original size; _attach_img_shapes:
    per-image img_shape tensor only when some image is smaller than the batch, stale attachments are removed."""
    from rsprompter_b200.detectors import _SamDetectorBase as D
    from rsprompter_b200.registry import make_data_samples
    x = torch.zeros(3, 3, 64, 96)
    ds = make_data_samples(3, (64, 96))
    ds[1].set_metainfo(dict(ori_shape=(40, 50), img_shape=(51, 64), scale_factor=(1.28, 1.275)))
    ds[2].set_metainfo(dict(ori_shape=(100, 200), img_shape=(64, 96), scale_factor=(2.0, 2.0)))
    hw, metas = D._metas(ds, x)
    assert hw == (64, 96) and metas[0] is None
    assert metas[1] == dict(ori_hw=(40, 50), crop_hw=(int(40 * 1.275), int(50 * 1.28)), scale_factor=(1.28, 1.275))
    assert metas[2]["crop_hw"] == (64, 96)                               # capped at the batch shape
    y = D._attach_img_shapes(ds, x)
    assert y is x and x.rsp_img_shapes.tolist() == [[64.0, 96.0], [51.0, 64.0], [64.0, 96.0]]
    D._attach_img_shapes(make_data_samples(3, (64, 96)), x)
    assert not hasattr(x, "rsp_img_shapes")
