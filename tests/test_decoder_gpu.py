"""SAM mask decoder on the H100 kernels vs the CPU oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(h, n_img, n_prompt, seed):
    from rsprompter_b200 import synthetic
    from rsprompter_b200.sam_config import SamDecoderArch
    from rsprompter_b200.sam_decoder import SamMaskDecoderB200
    arch = SamDecoderArch()
    sd = synthetic.mask_decoder_state_dict(arch, seed=seed)
    g = torch.Generator().manual_seed(seed)
    emb = torch.randn(n_img, 256, h, h, generator=g)
    pe = torch.randn(1, 256, h, h, generator=g)
    sparse = torch.randn(n_prompt, 1, 5, 256, generator=g)
    dec = SamMaskDecoderB200(arch)
    dec.load_state_dict(sd)
    return arch, sd, emb, pe, sparse, dec.cuda(), g


def _rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous()


@pytest.mark.parametrize("h,multimask", [(64, False), (32, False), (64, True)])
def test_shared_embedding_decode_matches_oracle(h, multimask):
    """Anchor-head calling pattern (M:1676-1694): broadcast no_mask_embed, prompts share images."""
    from oracle import restate
    arch, sd, emb, pe, sparse, dec, g = _setup(h, 2, 7, 21)
    prompt_img = torch.tensor([0, 0, 0, 1, 1, 1, 1], dtype=torch.int32)
    no_mask = torch.randn(256, generator=g)
    emb_pp = emb[prompt_img.long()]
    dense = no_mask.view(1, -1, 1, 1).expand(7, -1, h, h)
    m_ref, iou_ref = restate.mask_decoder(sd, arch, emb_pp, pe.expand(7, -1, -1, -1), sparse, dense, multimask)
    masks, iou = dec.decode(_rows(emb).cuda(), _rows(pe).cuda(), sparse[:, 0].cuda(), (h, h),
                            prompt_img=prompt_img.cuda(), dense_vec=no_mask.cuda(),
                            multimask_output=multimask)
    torch.cuda.synchronize()
    m_ref = m_ref[:, 0]
    assert masks.shape == m_ref.shape
    scale = max(1.0, m_ref.abs().max().item())
    err = (masks.cpu() - m_ref).abs().max().item()
    assert err < 2e-2 * scale, f"mask logits max abs err {err} (scale {scale})"
    assert (iou.cpu() - iou_ref[:, 0]).abs().max().item() < 2e-2 * max(1.0, iou_ref.abs().max().item())


def test_reference_signature_with_dense_prompts():
    """Query-head calling pattern (M:359-378): per-prompt dense embeddings, reference signature."""
    from oracle import restate
    from rsprompter_b200.registry import MODELS
    h = 32
    arch, sd, emb, pe, sparse, _, g = _setup(h, 4, 4, 22)
    dense = torch.randn(4, 256, h, h, generator=g)
    mod = MODELS.build(dict(type="RSSamMaskDecoder", hf_pretrain_name="facebook/sam-vit-base"))
    mod.mask_decoder.load_state_dict(sd)
    mod = mod.cuda()
    out = mod(image_embeddings=emb.cuda(), image_positional_embeddings=pe.expand(4, -1, -1, -1).cuda(),
              sparse_prompt_embeddings=sparse.cuda(), dense_prompt_embeddings=dense.cuda(),
              multimask_output=False, attention_similarity=None, target_embedding=None,
              output_attentions=None)
    assert len(out) == 3 and out[2] is None
    m_ref, iou_ref = restate.mask_decoder(sd, arch, emb, pe.expand(4, -1, -1, -1), sparse, dense, False)
    assert out[0].shape == m_ref.shape == (4, 1, 1, 4 * h, 4 * h) and out[1].shape == iou_ref.shape
    scale = max(1.0, m_ref.abs().max().item())
    assert (out[0].cpu() - m_ref).abs().max().item() < 2e-2 * scale
