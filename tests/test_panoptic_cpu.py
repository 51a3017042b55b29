"""Panoptic output of the query detectors without a GPU: the plain-torch restatement (oracle/restate_panoptic.py)
against the reference's own panoptic_postprocess and RSMaskFormerFusionHead.predict (tests/golden/reference_panoptic.pt,
made by tests/golden/make_golden_panoptic.py); what the fixture's adversarial cases exercise; how predict() follows
panoptic_on / instance_on / semantic_on; the bounds refused before any device work; what ptxas made of the kernels."""
import os
import re
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate_panoptic as rp  # noqa: E402

FX = torch.load(os.path.join(ROOT, "tests", "golden", "reference_panoptic.pt"), weights_only=False)
C, THINGS = FX["num_classes"], FX["num_things_classes"]


@pytest.mark.parametrize("name", sorted(FX["cases"]))
def test_oracle_equals_reference_panoptic_postprocess(name):
    case = FX["cases"][name]
    pan = rp.panoptic_postprocess(FX["mask_cls"], FX["mask_pred"], C, THINGS, case["test_cfg"])
    assert pan.dtype == torch.int32 and pan.shape == (1, 24, 32)
    assert torch.equal(pan, case["pan"])


@pytest.mark.parametrize("rescale,flt", [(True, False), (True, True), (False, False), (False, True)])
def test_oracle_equals_reference_fusion_predict(rescale, flt):
    p = FX["predict"]
    run = p["runs"][(rescale, flt)]
    out = rp.fusion_predict(p["mask_cls"][None], p["mask_pred"][None], [p["meta"]], C, THINGS, run["test_cfg"],
                            rescale=rescale)
    assert set(out[0]) == {"pan_results"}
    assert torch.equal(out[0]["pan_results"], run["pan"])
    # the same maps from the low-res logits through the resampling the detectors fuse into the kernel
    m = dict(ori_hw=(30, 40), crop_hw=(45, 60))
    up = rp.resample(p["logits"], (48, 64), dict(p["meta"]), rescale=rescale)
    pan = rp.panoptic_postprocess(p["mask_cls"], up, C, THINGS, run["test_cfg"])
    assert torch.equal(pan, run["pan"]) and pan.shape[1:] == (m["ori_hw"] if rescale else m["crop_hw"])


def _stats(name):
    return rp.panoptic_postprocess(FX["mask_cls"], FX["mask_pred"], C, THINGS, FX["cases"][name]["test_cfg"],
                                   stats=True)


def test_fixture_covers_the_adversarial_cases():
    pan, st = _stats("ties")
    by_q = {q: (ma, oa, sid) for q, ma, oa, sid in zip(st["query"], st["mask_area"], st["original_area"],
                                                       st["segment_id"])}
    assert 11 not in by_q                                            # argmax on the no-object class
    assert by_q[0][1] == 0 and by_q[0][2] == -1                      # the absorber: original_area 0, skipped
    assert by_q[1][:2] == (16, 16) and by_q[2][:2] == (32, 48)       # equal prob: the lower index wins
    assert (pan[0, 2:6, 2:6] == by_q[1][2]).all()
    pan, st = _stats("iou_exact")
    by_q = {q: (ma, oa, sid) for q, ma, oa, sid in zip(st["query"], st["mask_area"], st["original_area"],
                                                       st["segment_id"])}
    assert by_q[3][:2] == (6, 8) and by_q[3][2] >= 0                 # mask / original == iou_thr: kept
    assert by_q[5][:2] == (3, 5) and by_q[5][2] == -1                # below: skipped
    assert by_q[8][0] == 0 and by_q[8][1] == 8 and by_q[8][2] == -1   # mask_area 0: no instance id used
    things = [sid for sid in st["segment_id"] if sid >= 1000]
    assert sorted(s // 1000 for s in things) == list(range(1, len(things) + 1))
    assert by_q[6][2] == by_q[7][2] == 3                             # two stuff regions of one class
    assert by_q[10][1] == 16                                         # logits 0.0 and -1e-8 (not -1e-6): sigmoid 0.5
    assert 13 not in _stats("score_equals_thr")[1]["query"]        # score == object_mask_thr: dropped
    assert 13 in _stats("score_below_thr")[1]["query"]
    flt = FX["cases"]["filter_low_score"]["pan"]
    sid12 = by_q[12][2]
    assert (pan == sid12).sum() == 70 and (flt == sid12).sum() == 30
    assert (FX["cases"]["none_kept"]["pan"] == C).all()


def test_fixture_predict_runs_write_segments():
    for (rescale, _), run in FX["predict"]["runs"].items():
        assert run["pan"].shape == ((1, 30, 40) if rescale else (1, 45, 60))
        assert (run["pan"] != C).any() and (run["pan"] == C).any()


# ------------------------------------------------------------------------------ predict() flag handling
class _FakeFusionHead:
    num_classes, num_things_classes, num_stuff_classes = 5, 5, 0

    def __init__(self):
        self.calls = []

    def instance_postprocess_batched(self, cls, mask_pred, hw, metas=None, rescale=True):
        self.calls.append("instance")
        B = cls.shape[0]
        return dict(bboxes=torch.zeros(B, 1, 4), scores=torch.zeros(B, 1), labels=torch.zeros(B, 1, dtype=torch.long),
                    masks=torch.zeros(B, 1, *hw, dtype=torch.bool), is_thing=torch.ones(B, 1, dtype=torch.bool))

    def panoptic_postprocess_batched(self, cls, mask_pred, hw, metas=None, rescale=True):
        self.calls.append("panoptic")
        return [torch.full((1, *hw), 5, dtype=torch.int32) for _ in range(cls.shape[0])], None


def _predict(test_cfg, nq=4, num_classes=5):
    from rsprompter_b200.detectors import RSPrompterQuery, _SamDetectorBase
    from rsprompter_b200.registry import ConfigDict
    fh = _FakeFusionHead()
    fh.num_classes = num_classes
    raw_calls = []

    def raw(x):
        raw_calls.append(1)
        return dict(cls=torch.zeros(x.shape[0], nq, 6), mask_logits=torch.zeros(x.shape[0] * nq, 4, 4))

    self_ = SimpleNamespace(test_cfg=ConfigDict(test_cfg), panoptic_fusion_head=fh,
                            panoptic_head=SimpleNamespace(num_queries=nq), _raw=raw, _metas=_SamDetectorBase._metas,
                            _rle_masks=_SamDetectorBase._rle_masks)
    out = RSPrompterQuery.predict(self_, torch.zeros(2, 3, 16, 16))
    return out, fh.calls, raw_calls


def test_predict_defaults_to_panoptic_only():
    out, calls, _ = _predict(dict())
    assert calls == ["panoptic"]
    for ds in out:
        assert "pred_instances" not in ds and ds.pred_panoptic_seg.sem_seg.shape == (1, 16, 16)
        assert ds.pred_panoptic_seg.sem_seg.dtype == torch.int32


def test_predict_both_and_neither():
    out, calls, _ = _predict(dict(panoptic_on=True, instance_on=True, rle_masks=False))
    assert calls == ["instance", "panoptic"]
    assert all("pred_instances" in ds and "pred_panoptic_seg" in ds for ds in out)
    out, calls, _ = _predict(dict(panoptic_on=False, instance_on=True))
    assert calls == ["instance"] and all("pred_panoptic_seg" not in ds for ds in out)
    out, calls, _ = _predict(dict(panoptic_on=False, instance_on=False, rle_masks=True))
    assert calls == [] and all("pred_panoptic_seg" not in ds and "pred_instances" not in ds for ds in out)


def test_predict_refuses_semantic_output():
    for cfg in (dict(semantic_on=True), dict(panoptic_on=False, instance_on=True, semantic_on=True)):
        with pytest.raises(NotImplementedError):
            _predict(cfg)


@pytest.mark.parametrize("nq,num_classes", [(65536, 5), (4, 1000), (4, 0)])
def test_bounds_refused_before_device_work(nq, num_classes):
    with pytest.raises(ValueError):
        _predict(dict(), nq=nq, num_classes=num_classes)
    from rsprompter_b200.query_heads import RSMaskFormerFusionHead
    head = RSMaskFormerFusionHead(num_things_classes=min(num_classes, 3), num_stuff_classes=num_classes - min(num_classes, 3))
    with pytest.raises(ValueError):        # CPU tensors: any device work would raise RspError instead
        head.panoptic_postprocess_batched(torch.zeros(1, nq, num_classes + 1), torch.zeros(nq, 4, 4), (16, 16))


def test_bounds_accept_the_limits():
    from rsprompter_b200 import _lib
    _lib.check_panoptic_bounds(65535, 999)
    _, calls, raw_calls = _predict(dict(), nq=65535, num_classes=999)
    assert calls == ["panoptic"] and raw_calls == [1]


def test_pixel_data_work_alike():
    from rsprompter_b200.registry import HAVE_MMENGINE, PixelData
    p = PixelData(sem_seg=torch.ones(1, 2, 3, dtype=torch.int32))
    assert "sem_seg" in p and list(p.keys()) == ["sem_seg"]
    q = p.cpu()
    assert torch.equal(q.sem_seg, p.sem_seg) and q.to(torch.float32).sem_seg.dtype == torch.float32
    if HAVE_MMENGINE:   # pragma: no cover - mmengine is not installed here
        import mmengine.structures
        assert PixelData is mmengine.structures.PixelData


# ------------------------------------------------------------------------------ ptxas
def test_panoptic_kernels_do_not_spill():
    import __graft_entry__
    __graft_entry__.build()
    with open(os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "query.ptxas.log")) as f:
        log = f.read()
    entry = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
    spills = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    regs = re.compile(r"Used (\d+) registers")
    found, cur, sp = {}, None, None
    for line in log.splitlines():
        m = entry.search(line)
        if m:
            cur, sp = (m.group(1) if "panoptic" in m.group(1) else None), None
            continue
        if cur is None:
            continue
        m = spills.search(line)
        if m:
            sp = (int(m.group(1)), int(m.group(2)))
        m = regs.search(line)
        if m:
            found[cur] = (int(m.group(1)), sp)
            cur = None
    kinds = {k: v for k, v in found.items()}
    assert len(kinds) == 4, sorted(kinds)       # argmax (one resize, two resizes), decide, write
    for name, (r, sp) in kinds.items():
        assert sp == (0, 0), f"{name}: spill (store, load) bytes {sp}"
        assert r <= 128, f"{name}: {r} registers (256-thread blocks need <= 128 for two blocks per SM)"
