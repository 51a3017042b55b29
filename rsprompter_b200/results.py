"""Fixed-size per-rank result records and their cross-rank gather.

The inference path shards images across GPUs with no collective inside forward; the only exchange is ONE
all-gather of a compact result record after predict (the H100 counterpart of mmengine's ``collect_results`` after
``CocoMetric.process`` has encoded the masks, mmdet/evaluation/metrics/coco_metric.py:346-400, ``encode_mask_results``
:365).  A record is one flat byte buffer per rank holding, for its B images with M instance slots each:

    mask_bits  uint8  [B, M, H, W/8]   thresholded masks, bit-packed (pixel x = bit x % 8 of byte x // 8)
    rows       fp32   [B, M, 6]        x1, y1, x2, y2, score, label
    counts     int32  [B]              valid slots per image (slots >= count are padding)

The kernels write straight into views of the buffer (no packing pass); sections are 16-byte aligned."""
from __future__ import annotations

import torch
import torch.distributed as dist


def _align16(n: int) -> int:
    return (n + 15) // 16 * 16


class ResultRecord:
    def __init__(self, batch: int, slots: int, hw: tuple, device=None, buf: torch.Tensor | None = None):
        H, W = int(hw[0]), int(hw[1])
        assert W % 8 == 0, "record payload needs W % 8 == 0"
        self.batch, self.slots, self.hw = int(batch), int(slots), (H, W)
        nb = batch * slots * H * (W // 8)
        self._o_rows = _align16(nb)
        self._o_cnt = self._o_rows + _align16(batch * slots * 24)
        self.nbytes = self._o_cnt + _align16(batch * 4)
        if buf is None:
            buf = torch.zeros(self.nbytes, dtype=torch.uint8, device=device)
        assert buf.dtype == torch.uint8 and buf.is_contiguous() and buf.numel() == self.nbytes
        self.buf = buf
        self.mask_bits = buf[:nb].view(batch, slots, H, W // 8)
        self.rows = buf[self._o_rows:self._o_rows + batch * slots * 24].view(torch.float32).view(batch, slots, 6)
        self.counts = buf[self._o_cnt:self._o_cnt + batch * 4].view(torch.int32)

    def like(self, buf: torch.Tensor) -> "ResultRecord":
        """The same layout over another buffer (a gathered slice, a pinned host copy)."""
        return ResultRecord(self.batch, self.slots, self.hw, buf=buf)

    def gather(self, out: torch.Tensor | None = None, group=None) -> torch.Tensor:
        """The one collective of the path: uint8 [world, nbytes]; row r = rank r's record."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return self.buf.view(1, -1)
        world = dist.get_world_size(group)
        if out is None:
            out = torch.empty(world, self.nbytes, dtype=torch.uint8, device=self.buf.device)
        dist.all_gather_into_tensor(out.view(-1), self.buf, group=group)
        return out

    def split(self, gathered: torch.Tensor) -> list:
        return [self.like(gathered[r]) for r in range(gathered.shape[0])]

    def to_host(self, host: torch.Tensor | None = None, non_blocking: bool = True) -> "ResultRecord":
        if host is None:
            host = torch.empty(self.nbytes, dtype=torch.uint8, pin_memory=self.buf.is_cuda)
        host.copy_(self.buf, non_blocking=non_blocking)
        return self.like(host)

    def instances(self) -> list:
        """Per image: dict(bboxes [n,4], scores [n], labels int64 [n], masks bool [n,H,W]) - masks unpacked on the
        device the record lives on (numpy.unpackbits(bitorder='little') semantics on the host)."""
        H, W = self.hw
        out = []
        for b, n in enumerate(self.counts.tolist()):
            bits = self.mask_bits[b, :n]
            if bits.is_cuda:
                from . import _lib
                masks = _lib.unpack_mask_bits(bits.contiguous(), W)
            else:
                import numpy as np
                masks = torch.from_numpy(np.unpackbits(bits.numpy(), axis=-1, bitorder="little")[..., :W].astype(bool))
            r = self.rows[b, :n]
            out.append(dict(bboxes=r[:, :4], scores=r[:, 4], labels=r[:, 5].long(), masks=masks))
        return out


# ---- consumer side: COCO run-length encoding of host records -----------------------------------------------------
# What CocoMetric.process does to every predicted mask before results are collected (coco_metric.py:365 ->
# mmdet/structures/mask/utils.py:38-53 encode_mask_results -> pycocotools mask_util.encode).  pycocotools is a third-party
# C extension absent from this image and from /root/reference; the two functions below restate its published format
# (maskApi.c rleEncode / rleToString / rleFrString: column-major runs starting with a run of zeros; counts written as
# 5-bit groups + continuation bit, offset 48, with every count from the fourth on stored as the difference to the count
# two places back).  Host-side numpy on the bit-packed payload - evaluation itself stays outside this package.  The
# device encoder (encode_mask_results, device records; csrc/rle.cu) is held to these bytes.
def mask_to_coco_rle(mask) -> dict:
    """bool / uint8 [H, W] (numpy or CPU tensor) -> {'size': [H, W], 'counts': bytes}."""
    import numpy as np
    m = np.asarray(mask.numpy() if isinstance(mask, torch.Tensor) else mask).astype(bool)
    h, w = m.shape
    flat = m.T.reshape(-1)                                   # column-major, as the C API walks the mask
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate(([0], change, [flat.size]))
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts                                # the first run counts zeros
    out = bytearray()
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            ch = x & 0x1F
            x >>= 5                                          # arithmetic shift (negative differences)
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(ch + 48)
    return dict(size=[int(h), int(w)], counts=bytes(out))


def coco_rle_to_mask(rle: dict):
    """Inverse of mask_to_coco_rle -> numpy bool [H, W]."""
    import numpy as np
    h, w = rle["size"]
    s = rle["counts"]
    s = s.encode() if isinstance(s, str) else s
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            ch = s[p] - 48
            x |= (ch & 0x1F) << (5 * k)
            more = bool(ch & 0x20)
            p += 1
            k += 1
            if not more and (ch & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    flat = np.zeros(h * w, dtype=bool)
    pos, val = 0, False
    for c in counts:
        if val:
            flat[pos:pos + c] = True
        pos += c
        val = not val
    return flat.reshape(w, h).T


def encode_mask_results(masks) -> list:
    """Device counterpart of mmdet's encode_mask_results (mmdet/structures/mask/utils.py:37-53, called from
    CocoMetric.process, coco_metric.py:365): CUDA bool / uint8 masks [n, H, W] -> one {'size': [H, W], 'counts': bytes}
    dict per mask, byte for byte what mask_to_coco_rle (pycocotools) gives.  A list of such tensors (sizes may differ,
    e.g. one per image at its ori_shape) is encoded in one batched call and gives one list per tensor.  Only the RLE
    strings leave the device."""
    from . import _lib
    single = isinstance(masks, torch.Tensor)
    group = [m.contiguous() for m in ([masks] if single else masks)]
    strs = _lib.mask_rle([(m, m.shape[-1]) for m in group], packed=False)
    out, p = [], 0
    for m in group:
        n, h, w = m.shape
        out.append([dict(size=[int(h), int(w)], counts=s) for s in strs[p:p + n]])
        p += n
    return out[0] if single else out


def record_to_coco_results(rec: "ResultRecord", image_ids: list, label_to_cat=None) -> list:
    """Record -> the 'segm' result dicts CocoMetric.results2json writes (coco_metric.py:237-262): one dict per valid
    slot with image_id, bbox (xywh), score, category_id and the RLE-encoded mask.  A device record is encoded from its
    bits on the GPU (only the RLE strings, rows and counts are copied to the host); a host record in numpy."""
    import numpy as np
    H, W = rec.hw
    counts = rec.counts.tolist()
    rows = rec.rows.cpu().numpy()
    if rec.buf.is_cuda:
        from . import _lib
        strs = iter(_lib.mask_rle([(rec.mask_bits[b, :n], W) for b, n in enumerate(counts)], packed=True))
        segm = [[dict(size=[int(H), int(W)], counts=next(strs)) for _ in range(n)] for n in counts]
    else:
        bits = rec.mask_bits.numpy()
        masks = [np.unpackbits(bits[b, :n], axis=-1, bitorder="little")[..., :W].astype(bool) for b, n in enumerate(counts)]
        segm = [[mask_to_coco_rle(m) for m in mk] for mk in masks]
    out = []
    for b, n in enumerate(counts):
        for j in range(n):
            x1, y1, x2, y2, score, label = rows[b, j].tolist()
            cat = int(label) if label_to_cat is None else label_to_cat[int(label)]
            out.append(dict(image_id=image_ids[b], bbox=[x1, y1, x2 - x1, y2 - y1], score=float(score), category_id=cat,
                            segmentation=segm[b][j]))
    return out


# ---- mask polygons ------------------------------------------------------------------------------------------------
# What mmdet's DetLocalVisualizer does to every drawn mask: mmdet.structures.mask.bitmap_to_polygon
# (mmdet/structures/mask/structures.py:1166-1194), cv2.findContours(RETR_CCOMP, CHAIN_APPROX_NONE) per mask on the host.
# csrc/contours.cu computes the same contours on the device from the bit-packed masks; only the points are copied.
def _polygons_from_bits(groups: list, approx: int) -> list:
    """groups = [(bits uint8 [n, H, ceil(W/8)], W)] -> per mask (contours, hierarchy) in group order."""
    from . import _lib
    groups = [(b.contiguous(), int(W)) for b, W in groups if b.shape[0] > 0]
    if not groups:
        return []
    canvases = []
    for si, (b, W) in enumerate(groups):
        n, H, ld = b.shape
        canvases += [(H, W, [(si, j * H * ld, ld, H, H, W, 0, 0)]) for j in range(n)]
    return _lib.mask_contours([b for b, _ in groups], canvases, approx)


def _with_hole(contours, hierarchy):
    if hierarchy is None:
        return [], False
    return contours, bool((hierarchy.reshape(-1, 4)[:, 3] >= 0).any())


def bitmap_to_polygon(masks: torch.Tensor) -> list:
    """Device counterpart of mmdet's bitmap_to_polygon for a batch: CUDA bool / uint8 masks [n, H, W] (nonzero = set)
    -> one (contours, with_hole) per mask, contours int32 [k, 2] (x, y) arrays, exactly what the mmdet function returns
    for that mask.  The masks are bit-packed and traced on the GPU in one call."""
    from . import _lib
    m = masks.contiguous()
    if m.dtype == torch.uint8:
        m = m != 0
    return [_with_hole(c, h) for c, h in _polygons_from_bits([(_lib.pack_mask_bits(m), m.shape[-1])],
                                                             _lib.CHAIN_APPROX_NONE)]


def record_polygons(rec: "ResultRecord") -> list:
    """Per image of a device record, one (contours, with_hole) per valid slot: bitmap_to_polygon of its masks, traced
    from the record's bits."""
    from . import _lib
    W = rec.hw[1]
    counts = rec.counts.tolist()
    polys = iter(_polygons_from_bits([(rec.mask_bits[b, :n], W) for b, n in enumerate(counts)], _lib.CHAIN_APPROX_NONE))
    return [[_with_hole(*next(polys)) for _ in range(n)] for n in counts]


# ---- round-1 helpers kept for callers that only exchange the detection rows -------------------------------------
def pack_records(bboxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """[B,M,4], [B,M], [B,M] -> fp32 [B, M, 6]."""
    return torch.cat([bboxes.float(), scores.float()[..., None], labels.float()[..., None]], dim=2).contiguous()


def gather_records(records: torch.Tensor, counts: torch.Tensor):
    """All-gather [B, M, 6] rows with the int32 [B] counts appended, in one collective."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return records, counts
    world = dist.get_world_size()
    B = records.shape[0]
    flat = torch.cat([records.reshape(-1), counts.view(torch.float32).reshape(-1)])
    out = torch.empty(world, flat.numel(), dtype=flat.dtype, device=flat.device)
    dist.all_gather_into_tensor(out.view(-1), flat)
    n = records.numel()
    rec = out[:, :n].reshape((world * B,) + tuple(records.shape[1:]))
    cnt = out[:, n:].contiguous().view(torch.int32).reshape(world * B)
    return rec, cnt


def gather_mask_logits(mask_logits: torch.Tensor) -> torch.Tensor:
    """Alternative payload (SURVEY 8e): the low-resolution mask logits [B*M, h, w] as fp16, gathered over the default
    process group; the consumer resizes / thresholds them.  100 x 256^2 fp16 = 13 MB per image."""
    x = mask_logits.to(torch.float16).contiguous()
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return x
    out = torch.empty((dist.get_world_size() * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out, x)
    return out


def unpack_records(records: torch.Tensor, counts: torch.Tensor) -> list:
    out = []
    for r, n in zip(records, counts.tolist()):
        out.append(dict(bboxes=r[:n, :4], scores=r[:n, 4], labels=r[:n, 5].long()))
    return out
