"""The keep-ratio Resize + Pad rule (oracle.restate_resize) against mmcv's worked sizes and cv2.resize, and the
DetDataPreprocessor(device_transforms=...) configuration surface.  No GPU needed."""
import os
import re

import numpy as np
import pytest

from oracle import restate_resize as oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (h, w) -> (new_h, new_w) at scale (1024, 1024): mmcv rescale_size with _scale_size's + 0.5
WORKED = [((333, 500), (682, 1024)), ((600, 800), (768, 1024)), ((1000, 999), (1024, 1023)),
          ((3000, 1000), (1024, 341)), ((7, 3), (1024, 439)), ((1, 5), (205, 1024)), ((1024, 700), (1024, 700))]

CROP = (1024, 1024)
PAD = (0.406 * 255, 0.456 * 255, 0.485 * 255)
RESIZE = dict(type="Resize", scale=CROP, keep_ratio=True)
PAD_T = dict(type="Pad", size=CROP, pad_val=dict(img=PAD, masks=0))
DP = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], bgr_to_rgb=True, pad_size_divisor=32)


@pytest.mark.parametrize("hw, new", WORKED, ids=[f"{h}x{w}" for (h, w), _ in WORKED])
def test_rescale_size_worked_examples(hw, new):
    from rsprompter_b200.preprocess import rescale_size
    assert oracle.rescale_size(hw, CROP) == new
    assert rescale_size(hw, CROP) == new
    assert oracle.rescale_size(hw, (512, 512)) == rescale_size(hw, (512, 512))


def test_resize_metainfo():
    from rsprompter_b200.preprocess import resize_metainfo
    m = resize_metainfo((333, 500), (682, 1024), (1024, 1024))
    assert m == dict(ori_shape=(333, 500), scale_factor=(1024 / 500, 682 / 333), img_shape=(1024, 1024))
    _, om = oracle.resize_pad(np.zeros((333, 500, 3), np.uint8), CROP, CROP, PAD)
    assert om == m


@pytest.mark.parametrize("hw", [h for h, _ in WORKED] + [(512, 512), (2048, 2048), (2048, 1536)],
                         ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_resample_matches_cv2(hw):
    """The oracle's resample against cv2.resize(float32, INTER_LINEAR) on noise: a half-pixel or border error moves
    noise by tens of grey levels; IPP builds differ from the plain rule by < 0.01."""
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(hw[0] * 7 + hw[1]).integers(0, 256, (*hw, 3), dtype=np.uint8)
    new = oracle.rescale_size(hw, CROP)
    ref = cv2.resize(img.astype(np.float32), (new[1], new[0]), interpolation=cv2.INTER_LINEAR)
    got = oracle.resample(img, new)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 0.02


def test_pipeline_pads_with_the_normalised_pad_value():
    imgs = [np.full((300, 400, 3), 7, np.uint8)]
    x, metas = oracle.pipeline(imgs, CROP, CROP, PAD, DP["mean"], DP["std"])
    assert x.shape == (1, 3, 1024, 1024)
    assert metas[0]["img_shape"] == metas[0]["pad_shape"] == metas[0]["batch_input_shape"] == (1024, 1024)
    assert np.abs(x[0, :, 800:, :]).max() < 1e-6          # pad_val = the mean, in BGR
    np.testing.assert_allclose(x[0, :, 0, 0], (7 - np.array(DP["mean"])) / np.array(DP["std"]))


def _dp(**kw):
    from rsprompter_b200.preprocess import DetDataPreprocessor
    return DetDataPreprocessor(**dict(DP, **kw))


def test_device_transforms_accept_the_test_pipeline_dicts():
    dp = _dp(device_transforms=[RESIZE, PAD_T])
    scale, hw, pad = dp.device_transforms
    assert scale == CROP and hw == (1024, 1024) and pad == PAD
    dp = _dp(device_transforms=[dict(RESIZE, scale=(512, 512)), dict(PAD_T, size=(512, 512))])
    assert dp.device_transforms[1] == (512, 512)
    assert _dp().device_transforms is None                  # default off


def _reference_transforms():
    """Resize / Pad dicts of the test pipelines in an RSPrompter checkout's configs/rsprompter (named by the
    RSPROMPTER_ROOT environment variable), each evaluated with the file's crop_size."""
    base = os.environ.get("RSPROMPTER_ROOT")
    d = os.path.join(base, "configs", "rsprompter") if base else None
    if not d or not os.path.isdir(d):
        pytest.skip("RSPROMPTER_ROOT does not name an RSPrompter checkout with configs/rsprompter")
    out = []
    for sub in ("", "_base_"):
        for name in sorted(os.listdir(os.path.join(d, sub))):
            if not name.endswith(".py"):
                continue
            text = open(os.path.join(d, sub, name)).read()
            m = re.search(r"^crop_size\s*=\s*\((\d+),\s*(\d+)\)", text, flags=re.M)
            start = text.find("test_pipeline = [")
            if m is None or start < 0:
                continue
            body = text[start:text.index("\n]", start)]
            crop_size = (int(m.group(1)), int(m.group(2)))
            steps = [eval(line.strip().rstrip(","), {"dict": dict, "crop_size": crop_size})  # noqa: S307
                     for line in body.splitlines() if re.match(r"\s*dict\(type='(Resize|Pad)'", line)]
            if steps:
                out.append((os.path.join(sub, name), crop_size, steps))
    if not out:
        pytest.skip("no test pipeline with Resize + Pad found")
    return out


def test_device_transforms_accept_the_reference_configs():
    for name, crop_size, steps in _reference_transforms():
        dp = _dp(device_transforms=steps)
        scale, hw, pad = dp.device_transforms
        assert hw == (crop_size[1], crop_size[0]), name
        assert pad == PAD, name


@pytest.mark.parametrize("transforms, match", [
    ([dict(RESIZE, keep_ratio=False), PAD_T], "keep_ratio"),
    ([dict(RESIZE, type="RandomResize"), PAD_T], "exactly"),
    ([RESIZE], "exactly"),
    ([PAD_T, RESIZE], "exactly"),
    ([RESIZE, dict(type="Pad", size_divisor=32)], "size"),
    ([RESIZE, dict(PAD_T, pad_to_square=True)], "size"),
    ([dict(type="Resize", scale_factor=2.0, keep_ratio=True), PAD_T], "scale"),
    ([dict(RESIZE, interpolation="nearest"), PAD_T], "bilinear"),
    ([RESIZE, dict(PAD_T, size=(1000, 1000))], "pad_size_divisor"),
], ids=["keep_ratio_false", "other_type", "resize_only", "wrong_order", "size_divisor", "pad_to_square",
        "scale_factor", "nearest", "not_divisible"])
def test_device_transforms_reject_unsupported_forms(transforms, match):
    with pytest.raises(ValueError, match=match):
        _dp(device_transforms=transforms)


def test_device_transforms_reject_float_inputs():
    import torch
    dp = _dp(device_transforms=[RESIZE, PAD_T])
    with pytest.raises(ValueError, match="uint8"):
        dp(dict(inputs=[torch.zeros(3, 40, 50, dtype=torch.float32)]))


def test_header_declares_the_folded_resize_entry_points():
    from rsprompter_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "rsp_b200.h")).read()
    for name in ("rsp_resize_pad_u8", "rsp_mask_paste", "rsp_query_postprocess"):
        assert re.search(r"\bint\s+" + name + r"\s*\(", hdr), name
        assert name in _lib.declared_symbols()
    for name in ("rsp_mask_paste", "rsp_query_postprocess"):   # the rescale geometry and the record-slot bits
        proto = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", hdr).group(1)
        assert re.search(r"int Hb,\s*int Wb,\s*int crop_h,\s*int crop_w,\s*int H,\s*int W,\s*int Hr,\s*int Wr,\s*int packed",
                         proto), name
    assert re.search(r"#define\s+RSP_ABI_VERSION\s+3\b", hdr)
