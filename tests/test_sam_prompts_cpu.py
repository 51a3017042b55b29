"""SAM point / mask prompts without a GPU: the restatements of oracle.restate_prompts pinned to the HF modules on seeded
weights, the device path's own embed_points (plain tensor ops) against HF, RSSamPromptEncoder's parameter tree, every
shape rule that raises before device work, and what ptxas made of the multi-output upscale epilogue."""
import glob
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate, restate_prompts  # noqa: E402
from rsprompter_b200 import synthetic  # noqa: E402
from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch  # noqa: E402

LABELS = (1, 0, -1, -10, 2)


def _hf_config():
    from transformers import SamConfig
    cfg = SamConfig()
    cfg._attn_implementation = "eager"
    for sub in (cfg.vision_config, cfg.mask_decoder_config, cfg.prompt_encoder_config):
        sub._attn_implementation = "eager"
    return cfg


def _weights(seed=40):
    darch = SamDecoderArch()
    psd = synthetic.prompt_encoder_state_dict(darch, seed=seed)
    dsd = synthetic.mask_decoder_state_dict(darch, seed=seed + 1)
    gauss = synthetic.positional_embedding_state_dict(VISION_ARCHS["base"], seed + 2)["positional_embedding"]
    return darch, psd, dsd, gauss


@pytest.fixture(scope="module")
def hf_prompt_encoder():
    from transformers.models.sam.modeling_sam import SamPromptEncoder
    _, psd, _, gauss = _weights()
    m = SamPromptEncoder(_hf_config())
    m.load_state_dict(dict(psd, **{"shared_embedding.positional_embedding": gauss}), strict=True)
    return m.eval()


def _points(B, pb, n, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand(B, pb, n, 2, generator=g) * 1023
    lab = torch.tensor(LABELS)[torch.randint(0, len(LABELS), (B, pb, n), generator=g)]
    return pts, lab


@pytest.mark.parametrize("pad", [False, True])
def test_embed_points_restatement_matches_hf(hf_prompt_encoder, pad):
    _, psd, _, gauss = _weights()
    pts, lab = _points(2, 3, 7, seed=1)
    lab[0, 0, :5] = torch.tensor(LABELS)          # every label at least once
    with torch.no_grad():
        ref = hf_prompt_encoder._embed_points(pts, lab, pad)
    got = restate_prompts.embed_points(gauss, psd, pts, lab, pad, 1024)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("pad", [False, True])
def test_device_embed_points_matches_hf(hf_prompt_encoder, pad):
    """SamModelB200.embed_points is device tensor ops; on CPU tensors it runs here."""
    from rsprompter_b200.sam_model import SamModelB200
    _, psd, _, gauss = _weights()
    m = SamModelB200(VISION_ARCHS["base"], SamDecoderArch())
    m.prompt_encoder.load_state_dict(dict(psd, **{"shared_embedding.positional_embedding": gauss}), strict=True)
    pts, lab = _points(2, 4, 5, seed=2)
    lab[1, 1] = torch.tensor(LABELS)
    with torch.no_grad():
        ref = hf_prompt_encoder._embed_points(pts, lab, pad)
        got = m.embed_points(pts, lab, pad)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("case", ["points", "points_boxes", "masks", "nothing", "points_masks"])
def test_prompt_encoder_restatement_matches_hf(hf_prompt_encoder, case):
    _, psd, _, gauss = _weights()
    g = torch.Generator().manual_seed(3)
    pts, lab = _points(2, 3, 4, seed=4)
    boxes = torch.sort(torch.rand(2, 3, 4, generator=g) * 1000, dim=-1).values
    masks = torch.randn(2, 1, 256, 256, generator=g) * 4
    kw = dict(points=pts if "points" in case else None, labels=lab if "points" in case else None,
              boxes=boxes if "boxes" in case else None, masks=masks if "masks" in case else None)
    with torch.no_grad():
        rs, rd = hf_prompt_encoder(kw["points"], kw["labels"], kw["boxes"], kw["masks"])
    gs, gd = restate_prompts.prompt_encoder(gauss, psd, 1024, 64, **kw)
    assert (gs is None) == (rs is None)
    if rs is not None:
        torch.testing.assert_close(gs, rs, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(gd, rd, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("pb", [1, 3])
@pytest.mark.parametrize("multimask", [False, True])
def test_sam_model_forward_restatement_matches_hf(pb, multimask):
    """SamModel.forward(image_embeddings=...) with points (pb prompts per image) against prompt restatement ->
    restate_prompts.mask_decoder."""
    from transformers.models.sam.modeling_sam import SamModel
    darch, psd, dsd, gauss = _weights()
    hf = SamModel(_hf_config()).eval()
    sd = {"shared_image_embedding.positional_embedding": gauss,
          "prompt_encoder.shared_embedding.positional_embedding": gauss}
    sd.update({"prompt_encoder." + k: v for k, v in psd.items()})
    sd.update({"mask_decoder." + k: v for k, v in dsd.items()})
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("vision_encoder.") for k in missing)
    g = torch.Generator().manual_seed(5)
    emb = torch.randn(2, 256, 64, 64, generator=g)
    pts, lab = _points(2, pb, 2, seed=6)
    with torch.no_grad():
        out = hf(image_embeddings=emb, input_points=pts, input_labels=lab, multimask_output=multimask)
        sparse, dense = restate_prompts.prompt_encoder(gauss, psd, 1024, 64, points=pts, labels=lab)
        pe = restate.image_wide_positional_embedding(gauss, 64)
        m, iou = restate_prompts.mask_decoder(dsd, darch, emb, pe, sparse, dense, multimask)
    assert m.shape == out.pred_masks.shape and iou.shape == out.iou_scores.shape
    torch.testing.assert_close(m, out.pred_masks, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(iou, out.iou_scores, rtol=1e-4, atol=1e-4)


def _hf_prompt_encoder_names():
    from transformers.models.sam.modeling_sam import SamPromptEncoder
    return {k for k in SamPromptEncoder(_hf_config()).state_dict() if not k.startswith("shared_embedding.")}


def test_rssam_prompt_encoder_parameter_tree_and_strict_load(tmp_path):
    from rsprompter_b200.registry import MODELS
    pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base"))
    names = set(pe.prompt_encoder.state_dict())
    assert names == _hf_prompt_encoder_names()
    psd = synthetic.prompt_encoder_state_dict(seed=7)
    assert set(psd) == names
    # a trained RSPrompter-query checkpoint holds the module under ...prompt_encoder.prompt_encoder.
    ck = {"panoptic_head.prompt_encoder.prompt_encoder." + k: v for k, v in psd.items()}
    sub = {k[len("panoptic_head.prompt_encoder."):]: v for k, v in ck.items()}
    pe.load_state_dict(sub, strict=True)
    assert torch.equal(pe.prompt_encoder.not_a_point_embed.weight, psd["not_a_point_embed.weight"])
    assert torch.equal(pe.prompt_encoder.point_embed[3].weight, psd["point_embed.3.weight"])


def test_prompt_encoder_new_keys_leave_existing_weights_unchanged():
    """The point embeddings are drawn after the earlier tensors from the same generator."""
    gen = torch.Generator().manual_seed(2)
    first = torch.randn(1, 256, generator=gen) * 0.5
    assert torch.equal(synthetic.prompt_encoder_state_dict(seed=2)["no_mask_embed.weight"], first)


def test_rssam_prompt_encoder_no_mask_dense_on_cpu():
    from rsprompter_b200.registry import MODELS
    pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base"))
    pe.prompt_encoder.load_state_dict(synthetic.prompt_encoder_state_dict(seed=8), strict=True)
    sparse, dense = pe(None, None, None, None)
    assert sparse is None and dense.shape == (1, 256, 64, 64)
    assert torch.equal(dense[0, :, 3, 5], pe.prompt_encoder.no_mask_embed.weight[0])


# ---- every ValueError path, before any device work
@pytest.fixture(scope="module")
def cpu_model():
    from rsprompter_b200.sam_model import SamModelB200
    return SamModelB200(VISION_ARCHS["base"], SamDecoderArch())


EMB = torch.zeros(2, 256, 64, 64)


@pytest.mark.parametrize("kw, match", [
    (dict(input_points=torch.zeros(2, 3, 2)), "4D"),
    (dict(input_points=torch.zeros(2, 1, 3, 3)), r"\(x, y\)"),
    (dict(input_boxes=torch.zeros(2, 4)), "3D"),
    (dict(input_points=torch.zeros(2, 2, 1, 2), input_boxes=torch.zeros(2, 3, 4)), "as many bounding boxes"),
    (dict(input_points=torch.zeros(1, 1, 1, 2)), "batch size"),
    (dict(input_boxes=torch.zeros(3, 1, 4)), "batch size"),
    (dict(input_points=torch.zeros(2, 1, 2, 2), input_labels=torch.ones(2, 1, 3)), "input_labels"),
    (dict(input_masks=torch.zeros(2, 1, 64, 64)), "input_masks"),
    (dict(input_points=torch.zeros(2, 1, 11, 2)), "at most 11"),
    (dict(input_points=torch.zeros(2, 1, 10, 2), input_boxes=torch.zeros(2, 1, 4)), "at most 11"),
])
def test_sam_model_shape_rules_raise_before_device_work(cpu_model, kw, match):
    with pytest.raises(ValueError, match=match):
        cpu_model(image_embeddings=EMB, **kw)


def test_sam_model_token_bound_edge_passes_checks(cpu_model):
    """10 points + the pad point = 11 tokens is allowed: the checks pass and the call reaches the (CUDA-only) decoder."""
    assert cpu_model._check_prompts(2, torch.zeros(2, 1, 10, 2), None, None, None, 64) == (1, 11)
    assert cpu_model._check_prompts(2, torch.zeros(2, 5, 9, 2), None, torch.zeros(2, 5, 4), None, 64) == (5, 11)
    assert cpu_model._check_prompts(2, None, None, None, None, 64) == (1, 0)


def test_sam_model_image_source_rules(cpu_model):
    with pytest.raises(ValueError, match="Either"):
        cpu_model(input_points=torch.zeros(2, 1, 1, 2))
    with pytest.raises(ValueError, match="Only one"):
        cpu_model(pixel_values=torch.zeros(2, 3, 1024, 1024), image_embeddings=EMB)
    with pytest.raises(NotImplementedError):
        cpu_model(image_embeddings=EMB, attention_similarity=torch.zeros(1))


def test_get_prompt_embeddings_rules(cpu_model):
    with pytest.raises(ValueError, match="labels must also be provided"):
        cpu_model.get_prompt_embeddings(input_points=torch.zeros(1, 1, 1, 2))
    with pytest.raises(ValueError, match="at most 11"):
        cpu_model.get_prompt_embeddings(input_points=torch.zeros(1, 1, 12, 2), input_labels=torch.ones(1, 1, 12))


def test_prompt_encoder_and_decoder_modules_raise():
    from rsprompter_b200.registry import MODELS
    pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base"))
    with pytest.raises(ValueError, match="positional embedding"):
        pe(torch.zeros(1, 1, 1, 2), torch.ones(1, 1, 1), None, None)
    with pytest.raises(ValueError, match="positional embedding"):
        pe(None, None, torch.zeros(1, 1, 4), None)
    with pytest.raises(ValueError, match="input_masks"):
        pe(None, None, None, torch.zeros(1, 256, 256))
    dec = MODELS.build(dict(type="RSSamMaskDecoder", hf_pretrain_name="facebook/sam-vit-base"))
    pos = torch.zeros(1, 256, 64, 64)
    with pytest.raises(ValueError, match="at most 11"):
        dec(EMB, pos, torch.zeros(2, 3, 12, 256), torch.zeros(2, 256, 64, 64), False)
    with pytest.raises(ValueError, match="point_batch"):
        dec(EMB, pos, torch.zeros(3, 3, 2, 256), torch.zeros(2, 256, 64, 64), False)


def test_post_process_masks_rules():
    from rsprompter_b200.sam_model import post_process_masks
    with pytest.raises(ValueError, match="binarize"):
        post_process_masks([torch.zeros(1, 1, 256, 256)], [(600, 800)], [(768, 1024)], binarize=False)
    with pytest.raises(ValueError, match="one entry per image"):
        post_process_masks([torch.zeros(1, 1, 256, 256)], [(600, 800), (1, 1)], [(768, 1024)])


# ---- ptxas
BUILD = os.path.join(ROOT, "rsprompter_b200", "csrc", "build")
ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
HYPER = re.compile(r"_ZN3rsp2v225gemm_bf16_wgmma_v2_kernelILi128ELi([345])EEE")


def test_multi_output_upscale_does_not_spill():
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(BUILD, "gemm_v2.ptxas.log")) as f:
        text = f.read()
    assert "C7510" not in text
    spills, cur = {}, None
    for line in text.splitlines():
        m = ENTRY.search(line)
        if m:
            cur = m.group(1)
            continue
        m = SPILLS.search(line)
        if m and cur is not None:
            h = HYPER.search(cur)
            if h:
                spills[int(h.group(1))] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert set(spills) == {3, 4, 5}, spills          # 1, 2 and 3 outputs
    assert all(v == (0, 0) for v in spills.values()), spills
    assert glob.glob(os.path.join(BUILD, "*.ptxas.log"))
