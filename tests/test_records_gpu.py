"""Byte-level kernels either side of the path (SURVEY 8(f1), 8(f2)) on the GPU: bit-packed mask payload, the result
record, the uint8 DetDataPreprocessor kernels.  Integer / byte work: bit-exact."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]


@pytest.mark.parametrize("shape", [(3, 5, 64), (2, 7, 100), (1, 33, 1024), (4, 3, 37)])
def test_pack_unpack_bits_roundtrip(shape):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(shape[-1])
    m = torch.rand(*shape, generator=g) > 0.5
    bits = _lib.pack_mask_bits(m.cuda())
    ref = np.packbits(m.numpy(), axis=-1, bitorder="little")
    assert bits.shape == ref.shape and np.array_equal(bits.cpu().numpy(), ref)
    assert torch.equal(_lib.unpack_mask_bits(bits, shape[-1]).cpu(), m)


def test_mask_paste_into_bits_equals_packed_bytes():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(1)
    logits = (torch.randn(6, 64, 64, generator=g) * 3).cuda()
    for mode in (0, 1):
        thr = 0.5 if mode == 0 else 0.0
        ref = _lib.mask_paste(logits, thr, raw=mode == 1, size=(256, 256))
        bits = _lib.mask_paste(logits, thr, raw=mode == 1, bits=torch.empty(6, 256, 32, dtype=torch.uint8).cuda())
        assert bits.shape == (6, 256, 32)
        assert np.array_equal(bits.cpu().numpy(), np.packbits(ref.cpu().numpy(), axis=-1, bitorder="little"))


def test_query_postprocess_into_bits_equals_unpacked():
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(2)
    logits = (torch.randn(12, 64, 64, generator=g) * 2).cuda()
    sel = torch.tensor([3, 0, 11, 7, 7], dtype=torch.int32).cuda()
    sc = torch.rand(5, generator=g).cuda()
    masks, s0, b0 = _lib.query_postprocess(logits, sel, sc, (256, 256))
    bits, s1, b1 = _lib.query_postprocess(logits, sel, sc, bits=torch.empty(5, 256, 32, dtype=torch.uint8).cuda())
    assert torch.equal(s0, s1) and torch.equal(b0, b1)
    assert torch.equal(_lib.unpack_mask_bits(bits, 256), masks)


@pytest.mark.parametrize("swap", [True, False])
@pytest.mark.parametrize("hwc", [False, True])
def test_preprocess_u8_matches_torch(swap, hwc):
    """(x[channel flip] - mean) / std in fp32 with padding, bit-exact against the torch expression of
    mmengine ImgDataPreprocessor.forward / mmdet DetDataPreprocessor (data_preprocessor.py:110-148)."""
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(3)
    h, w, H, W = 45, 70, 64, 96
    img = torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8)
    src = img.cuda()
    if hwc:   # a decoded HWC array viewed as CHW (non-contiguous planes)
        src = img.permute(1, 2, 0).contiguous().cuda().permute(2, 0, 1)
    out = torch.empty(3, H, W, device="cuda")
    _lib.preprocess_u8(src, out, MEAN, STD, swap, 1.5)
    x = img[[2, 1, 0]] if swap else img
    ref = torch.full((3, H, W), 1.5)
    ref[:, :h, :w] = (x.float() - torch.tensor(MEAN).view(3, 1, 1)) / torch.tensor(STD).view(3, 1, 1)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("hwc", [False, True])
def test_patchify16_u8_equals_preprocess_then_patchify(hwc):
    from rsprompter_b200 import _lib
    g = torch.Generator().manual_seed(4)
    B, S = 2, 64
    img = torch.randint(0, 256, (B, 3, S, S), generator=g, dtype=torch.uint8).cuda()
    src = img.contiguous(memory_format=torch.channels_last) if hwc else img
    f = torch.empty(B, 3, S, S, device="cuda")
    for b in range(B):
        _lib.preprocess_u8(img[b], f[b], MEAN, STD, True, 0.0)
    ref = _lib.patchify16(f)
    got = _lib.patchify16_u8(src, MEAN, STD, True)
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))


def test_data_preprocessor_u8_paths():
    """DetDataPreprocessor on uint8 CHW inputs: kernel path == the float torch path; the fused hand-over keeps bytes."""
    from rsprompter_b200.registry import MODELS
    cfgd = dict(type="DetDataPreprocessor", mean=MEAN, std=STD, bgr_to_rgb=True, pad_size_divisor=32, pad_value=0)
    pre = MODELS.build(cfgd).cuda()
    g = torch.Generator().manual_seed(5)
    imgs = [torch.randint(0, 256, (3, 50, 64), generator=g, dtype=torch.uint8),
            torch.randint(0, 256, (3, 64, 40), generator=g, dtype=torch.uint8)]
    out = pre(dict(inputs=[t.clone() for t in imgs]), False)
    ref = pre(dict(inputs=[t.float() for t in imgs]), False)       # float inputs: round-1 torch expression
    assert out["inputs"].shape == (2, 3, 64, 64) and torch.equal(out["inputs"], ref["inputs"])
    assert out["data_samples"][0].metainfo["batch_input_shape"] == (64, 64)
    same = torch.randint(0, 256, (2, 3, 64, 64), generator=g, dtype=torch.uint8)
    fused = pre(dict(inputs=same), False, fuse_patch_embed=True)["inputs"]
    assert fused.dtype == torch.uint8 and fused.rsp_norm[2] is True and torch.equal(fused.cpu(), same)
