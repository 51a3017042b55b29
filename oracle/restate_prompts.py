"""fp32 CPU restatement of SAM's point / mask prompt path (TEST INFRASTRUCTURE, see oracle/__init__.py): HF
SamPromptEncoder._embed_points and forward, and SamMaskDecoder.forward with HF's [B, point_batch] layout.  Built from
the bricks of oracle.restate, which stays as it is.

Citations: HF: = transformers/models/sam/modeling_sam.py (5.5.0 copy in this image)."""
from __future__ import annotations

import math

import torch

from . import restate


def positional_embedding(gauss: torch.Tensor, coords: torch.Tensor, image_size: int) -> torch.Tensor:
    """SamPositionalEmbedding.forward (HF:552-566) on image-space coordinates [..., 2] normalised by image_size."""
    c = coords.clone()
    c[..., 0] = c[..., 0] / image_size
    c[..., 1] = c[..., 1] / image_size
    c = (2 * c - 1) @ gauss
    c = 2 * math.pi * c
    return torch.cat([torch.sin(c), torch.cos(c)], dim=-1)


def embed_points(gauss: torch.Tensor, psd: dict, points: torch.Tensor, labels: torch.Tensor, pad: bool,
                 image_size: int) -> torch.Tensor:
    """SamPromptEncoder._embed_points (HF:613-645): points [B, pb, n, 2], labels [B, pb, n] -> [B, pb, n (+1), C]."""
    points = points + 0.5
    labels = labels.to(torch.float32)
    if pad:
        points = torch.cat([points, torch.zeros(*points.shape[:2], 1, 2)], dim=2)
        labels = torch.cat([labels, -torch.ones(*labels.shape[:2], 1)], dim=2)
    emb = positional_embedding(gauss, points, image_size)
    out = emb.clone()
    for idx in torch.cartesian_prod(*[torch.arange(s) for s in labels.shape]).tolist():
        b, j, k = idx
        lab = labels[b, j, k].item()
        if lab == -1:
            out[b, j, k] = psd["not_a_point_embed.weight"][0]
        elif lab == -10:
            out[b, j, k] = 0.0
        elif lab == 0:
            out[b, j, k] = emb[b, j, k] + psd["point_embed.0.weight"][0]
        elif lab == 1:
            out[b, j, k] = emb[b, j, k] + psd["point_embed.1.weight"][0]
    return out


def prompt_encoder(gauss: torch.Tensor, psd: dict, image_size: int, grid: int, points=None, labels=None, boxes=None,
                   masks=None, eps: float = 1e-6):
    """SamPromptEncoder.forward (HF:658-698) -> (sparse [B, pb, P, C] or None, dense [B or 1, C, grid, grid])."""
    sparse = None
    batch = 1
    if points is not None:
        batch = points.shape[0]
        sparse = embed_points(gauss, psd, points, labels, boxes is None, image_size)
    if boxes is not None:
        batch = boxes.shape[0]
        be = restate.embed_boxes(gauss, psd["point_embed.2.weight"], psd["point_embed.3.weight"], boxes, image_size)
        sparse = be if sparse is None else torch.cat([sparse, be], dim=2)
    if masks is not None:
        dense = restate.sam_mask_embedding(psd, masks, eps)
    else:
        dense = psd["no_mask_embed.weight"].reshape(1, -1, 1, 1).expand(batch, -1, grid, grid)
    return sparse, dense


def mask_decoder(sd: dict, arch, image_embeddings: torch.Tensor, image_pe: torch.Tensor, sparse, dense: torch.Tensor,
                 multimask_output: bool):
    """SamMaskDecoder.forward (HF:461-543) in HF's layout: image_embeddings [B, C, h, w], image_pe [1 or B, C, h, w],
    sparse [B, pb, P, C] or None, dense [B or 1, C, h, w].  Each image's (embedding + dense) is repeated for its pb
    prompts (repeat_interleave, HF:499-501).  -> masks [B, pb, n_out, 4h, 4w], iou [B, pb, n_out]."""
    B, C, h, w = image_embeddings.shape
    if sparse is None:
        sparse = torch.zeros(B, 1, 0, C)
    pb = sparse.shape[1]
    src = (image_embeddings + dense).repeat_interleave(pb, 0)
    pe = image_pe.expand(B, -1, -1, -1).repeat_interleave(pb, 0)
    m, iou = restate.mask_decoder(sd, arch, src, pe, sparse.reshape(B * pb, 1, -1, C), torch.zeros(1, C, 1, 1),
                                  multimask_output)
    return m.reshape(B, pb, *m.shape[2:]), iou.reshape(B, pb, -1)
