"""SAM point and mask prompts on the GPU (ViT-B synthetic weights): RSSamModel with points, labels, boxes and mask
prompts against the fp32 restatement (restate.vit_encoder -> restate_prompts.prompt_encoder ->
restate_prompts.mask_decoder), the image_embeddings path, get_prompt_embeddings, RSSamPromptEncoder and
RSSamMaskDecoder with point_batch > 1, the multi-output upscale GEMM against single-output launches, and
post_process_masks.  Tolerances are those of test_samdet_box_prompted_sam_matches_oracle."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sam():
    from oracle import restate
    from rsprompter_b200 import synthetic
    from rsprompter_b200.registry import MODELS
    from rsprompter_b200.sam_config import VISION_ARCHS, SamDecoderArch
    arch, darch = VISION_ARCHS["base"], SamDecoderArch()
    vsd = synthetic.vision_encoder_state_dict(arch, seed=51)
    dsd = synthetic.mask_decoder_state_dict(darch, seed=52)
    psd = synthetic.prompt_encoder_state_dict(darch, seed=53)
    gauss = synthetic.positional_embedding_state_dict(arch, 54)["positional_embedding"]
    sd = {"shared_image_embedding.positional_embedding": gauss}
    sd.update({"vision_encoder." + k: v for k, v in vsd.items()})
    sd.update({"mask_decoder." + k: v for k, v in dsd.items()})
    sd.update({"prompt_encoder." + k: v for k, v in psd.items()})
    model = MODELS.build(dict(type="RSSamModel", hf_pretrain_name="facebook/sam-vit-base"))
    model.sam_model.load_state_dict(sd, strict=True)
    model = model.cuda()
    x = torch.randn(2, 3, 1024, 1024, generator=torch.Generator().manual_seed(55))
    with torch.no_grad():
        emb, _ = restate.vit_encoder(vsd, arch, x)
    pe = restate.image_wide_positional_embedding(gauss, 64)
    return dict(model=model, x=x, emb=emb, pe=pe, dsd=dsd, psd=psd, gauss=gauss, darch=darch)


def _prompts(case, seed):
    g = torch.Generator().manual_seed(seed)
    B = 2
    pb = {"single": 1, "mixed": 4, "pb16": 16, "points_box": 4, "mask": 1, "mask_points": 4, "nothing": 1}[case]
    n = {"single": 1, "mixed": 3, "pb16": 2, "points_box": 2, "mask_points": 2}.get(case, 0)
    kw = {}
    if n:
        kw["input_points"] = torch.rand(B, pb, n, 2, generator=g) * 1023
        if case == "mixed":
            kw["input_labels"] = torch.tensor([1, 0, -1, -10, 2])[torch.randint(0, 5, (B, pb, n), generator=g)]
            kw["input_labels"][0, 0] = torch.tensor([1, 0, -10])
        else:
            kw["input_labels"] = torch.randint(0, 2, (B, pb, n), generator=g)
    if case == "points_box":
        kw["input_boxes"] = torch.sort(torch.rand(B, pb, 4, generator=g) * 1000, dim=-1).values
    if case in ("mask", "mask_points"):
        kw["input_masks"] = torch.randn(B, 1, 256, 256, generator=g) * 4
    return kw


def _oracle(sam, kw, multimask):
    from oracle import restate_prompts
    with torch.no_grad():
        sparse, dense = restate_prompts.prompt_encoder(
            sam["gauss"], sam["psd"], 1024, 64, points=kw.get("input_points"), labels=kw.get("input_labels"),
            boxes=kw.get("input_boxes"), masks=kw.get("input_masks"))
        return restate_prompts.mask_decoder(sam["dsd"], sam["darch"], sam["emb"], sam["pe"], sparse, dense, multimask)


def _close(got_m, got_iou, ref_m, ref_iou):
    assert tuple(got_m.shape) == tuple(ref_m.shape) and tuple(got_iou.shape) == tuple(ref_iou.shape)
    err = (got_m.cpu() - ref_m).abs().max().item()
    assert err <= 2e-2 * max(1.0, ref_m.abs().max().item()), err
    assert (got_iou.cpu() - ref_iou).abs().max().item() <= 2e-2


@pytest.mark.parametrize("multimask", [False, True])
@pytest.mark.parametrize("case", ["single", "mixed", "pb16", "points_box", "mask", "mask_points", "nothing"])
def test_rssam_model_prompts_match_oracle(sam, case, multimask):
    kw = _prompts(case, seed=7 * len(case) + (3 if multimask else 0))
    model = sam["model"]
    out = model(pixel_values=sam["x"].cuda(), multimask_output=multimask,
                **{k: v.cuda() for k, v in kw.items()})
    torch.cuda.synchronize()
    ref_m, ref_iou = _oracle(sam, kw, multimask)
    _close(out.pred_masks, out.iou_scores, ref_m, ref_iou)
    # the interactive loop: encode once, then prompt the cached embeddings -- the same bytes
    emb = model.get_image_embeddings(sam["x"].cuda())
    assert emb.shape == (2, 256, 64, 64) and emb.dtype == torch.float32
    out2 = model(image_embeddings=emb, multimask_output=multimask, **{k: v.cuda() for k, v in kw.items()})
    assert torch.equal(out.pred_masks, out2.pred_masks) and torch.equal(out.iou_scores, out2.iou_scores)


def test_default_labels_are_ones(sam):
    kw = _prompts("mixed", seed=3)
    pts = kw["input_points"].cuda()
    a = sam["model"](pixel_values=sam["x"].cuda(), input_points=pts)
    b = sam["model"](pixel_values=sam["x"].cuda(), input_points=pts, input_labels=torch.ones(pts.shape[:3]).cuda())
    assert torch.equal(a.pred_masks, b.pred_masks) and a.pred_masks.shape[2] == 3     # multimask_output defaults on


@pytest.mark.parametrize("case", ["mixed", "points_box", "mask_points", "nothing"])
def test_get_prompt_embeddings_match_oracle(sam, case):
    from oracle import restate_prompts
    kw = _prompts(case, seed=7)
    sparse, dense = sam["model"].get_prompt_embeddings(**{k: v.cuda() for k, v in kw.items()})
    rs, rd = restate_prompts.prompt_encoder(sam["gauss"], sam["psd"], 1024, 64, points=kw.get("input_points"),
                                            labels=kw.get("input_labels"), boxes=kw.get("input_boxes"),
                                            masks=kw.get("input_masks"))
    assert (sparse is None) == (rs is None)
    if rs is not None:
        torch.testing.assert_close(sparse.cpu(), rs, rtol=1e-4, atol=1e-4)
    assert dense.shape[1:] == (256, 64, 64)
    torch.testing.assert_close(dense.cpu(), rd.expand(dense.shape[0], -1, -1, -1), rtol=1e-4, atol=1e-4)


def test_rssam_prompt_encoder_forward(sam):
    from oracle import restate
    from rsprompter_b200.registry import MODELS
    pe = MODELS.build(dict(type="RSSamPromptEncoder", hf_pretrain_name="facebook/sam-vit-base"))
    pe.prompt_encoder.load_state_dict(sam["psd"], strict=True)
    pe = pe.cuda()
    masks = torch.randn(3, 1, 256, 256, generator=torch.Generator().manual_seed(9)) * 4
    sparse, dense = pe(None, None, None, masks.cuda())
    ref = restate.sam_mask_embedding(sam["psd"], masks)
    assert sparse is None and dense.shape == (3, 256, 64, 64)
    torch.testing.assert_close(dense.cpu(), ref, rtol=1e-4, atol=1e-4)
    sparse, dense = pe(None, None, None, None)
    assert sparse is None and torch.equal(dense[0, :, 0, 0].cpu(), sam["psd"]["no_mask_embed.weight"][0])


@pytest.mark.parametrize("multimask", [False, True])
def test_rssam_mask_decoder_point_batch(sam, multimask):
    from oracle import restate_prompts
    from rsprompter_b200.registry import MODELS
    dec = MODELS.build(dict(type="RSSamMaskDecoder", hf_pretrain_name="facebook/sam-vit-base"))
    dec.mask_decoder.load_state_dict(sam["dsd"], strict=True)
    dec = dec.cuda()
    g = torch.Generator().manual_seed(11)
    sparse = torch.randn(2, 5, 3, 256, generator=g)
    dense = torch.randn(2, 256, 64, 64, generator=g) * 0.1
    m, iou, _ = dec(sam["emb"].cuda(), sam["pe"].cuda(), sparse.cuda(), dense.cuda(), multimask)
    ref_m, ref_iou = restate_prompts.mask_decoder(sam["dsd"], sam["darch"], sam["emb"], sam["pe"], sparse, dense,
                                                  multimask)
    _close(m, iou, ref_m, ref_iou)


@pytest.mark.parametrize("grid", [64, 32])
@pytest.mark.parametrize("n", [1, 7, 130])
def test_multi_output_upscale_equals_single_output_launches(n, grid):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(n * 100 + grid)
    up1 = (torch.randn(n * 4 * grid * grid, 64, generator=g)).to(torch.bfloat16).cuda()
    w = (torch.randn(128, 64, generator=g) * 0.2).to(torch.bfloat16).cuda()
    b = (torch.randn(128, generator=g) * 0.1).cuda()
    for n_out in (3, 2):
        hyper = torch.randn(n, n_out, 32, generator=g).cuda()
        fused = _lib.gemm_upscale_masks(up1, w, b, hyper, grid, grid)
        single = torch.stack([_lib.gemm_upscale_mask(up1, w, b, hyper[:, o].contiguous(), grid, grid)
                              for o in range(n_out)], dim=1)
        torch.cuda.synchronize()
        assert fused.shape == (n, n_out, 4 * grid, 4 * grid)
        assert torch.equal(fused, single)


def test_post_process_masks_matches_interpolate_chain():
    from rsprompter_b200.sam_model import post_process_masks
    g = torch.Generator().manual_seed(13)
    lows = [torch.randn(3, 3, 256, 256, generator=g) * 3, torch.randn(1, 1, 256, 256, generator=g) * 3]
    ori, rs = [(600, 800), (500, 333)], [(768, 1024), (1024, 682)]
    got = post_process_masks([m.cuda() for m in lows], ori, rs)
    for m, o, r, gm in zip(lows, ori, rs, got):
        x = F.interpolate(m, (1024, 1024), mode="bilinear", align_corners=False)[..., :r[0], :r[1]]
        x = F.interpolate(x, o, mode="bilinear", align_corners=False)
        assert gm.shape == x.shape and gm.dtype == torch.bool
        far = x.abs() > 1e-3
        assert torch.equal(gm.cpu()[far], (x > 0)[far])
