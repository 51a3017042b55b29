"""ctypes binding of ``librsp_b200.so`` (C ABI declared in ``include/rsp_b200.h``).

The product path has no CPU or eager-PyTorch fallback: if the shared library is missing the
import fails loudly, and every wrapper raises ``RspError`` on a non-zero status.  Tensors are
passed as raw device pointers; PyTorch is only the allocator and stream provider.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

import torch

_PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = _PKG_DIR / "librsp_b200.so"
CSRC_DIR = _PKG_DIR / "csrc"


class RspError(RuntimeError):
    """Raised when an ``rsp_*`` entry point returns a non-zero status."""


def build_library(verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a into ``librsp_b200.so`` (in-tree, via make)."""
    cmd = ["make", "-C", str(CSRC_DIR), "-j", str(os.cpu_count() or 4), "all"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"building librsp_b200.so failed:\n{res.stdout[-4000:]}\n{res.stderr[-4000:]}")
    if verbose:
        print(res.stdout[-2000:])
    return LIB_PATH


def _load() -> ctypes.CDLL:
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} not found: the CUDA extension is mandatory (no fallback path). "
            "Run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C rsprompter_b200/csrc`.")
    return ctypes.CDLL(str(LIB_PATH))


_lib = _load()

_vp, _i, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float

_SIGNATURES = {
    "rsp_abi_version": ([], _i),
    "rsp_last_error": ([], ctypes.c_char_p),
    "rsp_gemm_bf16": ([_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _vp], _i),
    "rsp_gemm_bf16_simt": ([_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _vp], _i),
    "rsp_vit_attention": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp], _i),
    "rsp_vit_attention_scatter": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp], _i),
    "rsp_vit_attention_simt": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp], _i),
    "rsp_layernorm": ([_vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _f, _i, _vp, _i, _vp], _i),
    "rsp_patchify16": ([_vp, _vp, _i, _i, _i, _vp], _i),
    "rsp_layernorm_add": ([_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, ctypes.c_longlong, _i, _f, _vp], _i),
    "rsp_im2col_nhwc": ([_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp], _i),
    "rsp_nhwc_to_nchw": ([_vp, _i, _vp, _i, _i, _i, _vp], _i),
    "rsp_cast_f32_bf16": ([_vp, _vp, ctypes.c_longlong, _vp], _i),
    "rsp_add_table_bf16": ([_vp, _vp, _vp, ctypes.c_longlong, ctypes.c_longlong, _vp], _i),
    "rsp_gemm_bf16_ex": ([_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i,
                          _i, _vp, _vp, _f, _vp, _i, _vp, _vp, _i, _i, _vp], _i),
    "rsp_add_cast_bf16": ([_vp, _vp, _vp, ctypes.c_longlong, ctypes.c_longlong, _vp], _i),
    "rsp_token_self_attention": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp], _i),
    "rsp_t2i_attention": ([_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp], _i),
    "rsp_i2t_attention": ([_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp], _i),
    "rsp_t2i_fused": ([_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp], _i),
    "rsp_i2t_fused": ([_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _vp], _i),
    "rsp_rpn_decode": ([_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _f, _f, _f, _i, _i, _vp, _vp, _vp], _i),
    "rsp_bbox_cls_decode": ([_vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _f, _f, _f, _vp, _vp, _vp, _vp], _i),
    "rsp_rpn_decode_shapes": ([_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _f, _i, _i, _vp, _vp, _vp], _i),
    "rsp_nms_batched_topk": ([_vp, _vp, _vp, _i, _i, _f, _vp, _vp, _vp, _i, _vp], _i),
    "rsp_bbox_cls_decode_shapes": ([_vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp], _i),
    "rsp_nms_batched": ([_vp, _vp, _vp, _i, _i, _f, _vp, _vp, _vp, _vp], _i),
    "rsp_compact_keep": ([_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp], _i),
    "rsp_soft_nms_workspace_bytes": ([_i, _i, _i, _vp], _i),
    "rsp_soft_nms_batched": ([_vp, _vp, _vp, _vp, _i, _i, _i, _f, _f, _f, _i, _i, _i, _vp, ctypes.c_size_t, _vp, _vp,
                              _vp, _vp, _vp, _vp], _i),
    "rsp_roi_align_nhwc": ([_vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _f, _vp, _vp], _i),
    "rsp_mask_paste": ([_vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp], _i),
    "rsp_pool2_nhwc": ([_vp, _vp, _i, _i, _i, _i, _i, _vp], _i),
    "rsp_zero_border_nhwc": ([_vp, _i, _i, _i, _i, _vp], _i),
    "rsp_sigmoid_f32": ([_vp, _vp, ctypes.c_longlong, _vp], _i),
    "rsp_mask_paste_boxes": ([_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp], _i),
    "rsp_groupnorm_nhwc": ([_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp], _i),
    "rsp_ms_deform_attn_sample": ([_vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp], _i),
    "rsp_mha_small": ([_vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp], _i),
    "rsp_ms_deform_attn_sample_c": ([_vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp], _i),
    "rsp_mha_small_hd": ([_vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _i, _vp], _i),
    "rsp_conv3x3_nhwc_bf16": ([_vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _i, _i, _i, _i, _vp], _i),
    "rsp_conv3x3_geometry_ok": ([_i, _i, _i, _i], _i),
    "rsp_mask_paste_rescale": ([_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, ctypes.c_float, _i, _vp], _i),
    "rsp_query_postprocess_rescale": ([_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp], _i),
    "rsp_attn_mask_bits": ([_vp, _i, _i, _i, _vp, _vp], _i),
    "rsp_resize_bilinear_nhwc": ([_vp, _i, _i, _i, _i, _i, _i, _vp, _vp], _i),
    "rsp_mask_embed_src": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp], _i),
    "rsp_query_postprocess": ([_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp], _i),
    "rsp_sin_fold": ([_vp, _vp, ctypes.c_longlong, _vp], _i),
    "rsp_attn_softmax_bias": ([_vp, _i, _vp, _i, _i, _vp, _i, _i, _i, _i, _f, _vp], _i),
    "rsp_transpose_cols": ([_vp, _i, _i, _i, _i, _i, _vp, _vp], _i),
    "rsp_split_heads": ([_vp, _i, _i, _i, _i, _i, _i, _vp, _vp], _i),
    "rsp_gemm_bf16_grouped": ([_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp], _i),
    "rsp_query_postprocess_bits": ([_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp], _i),
    "rsp_mask_paste_bits": ([_vp, _vp, _i, _i, _i, _f, _i, _vp], _i),
    "rsp_pack_mask_bits": ([_vp, _vp, ctypes.c_longlong, _i, _vp], _i),
    "rsp_unpack_mask_bits": ([_vp, _vp, ctypes.c_longlong, _i, _vp], _i),
    "rsp_preprocess_u8": ([_vp, _i, _i, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_longlong, _vp, _i, _i, _vp, _vp,
                           _i, _f, _vp], _i),
    "rsp_patchify16_u8": ([_vp, _i, _vp, _i, _i, _i, _vp, _vp, _i, _vp], _i),
    "rsp_resize_pad_u8": ([_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _i, _vp, _vp], _i),
    "rsp_mask_paste_rescale_bits": ([_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _i, _vp], _i),
    "rsp_query_postprocess_rescale_bits": ([_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp,
                                            _vp, _vp], _i),
    "rsp_mask_rle_lengths": ([_vp, _i, _vp, _vp, _i, _vp, _vp], _i),
    "rsp_mask_rle_write": ([_vp, _i, _vp, _i, _vp, _vp, _vp, _vp], _i),
    "rsp_mask_rle_placed_lengths": ([_vp, _i, _vp, _vp, _i, _vp, _vp], _i),
    "rsp_mask_rle_placed_write": ([_vp, _i, _vp, _i, _vp, _vp, _vp, _vp], _i),
    "rsp_gemm_upscale_masks": ([_vp, _i, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _i, _i, _vp], _i),
    "rsp_sam_mask_embed": ([_vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp], _i),
    "rsp_sam_mask_stats": ([_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _f, _f, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp,
                            _vp], _i),
    "rsp_sam_mask_stats_crop": ([_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _f, _f, _vp, _f, _f, _i, _i, _i, _i, _i,
                                 _i, _vp, _vp, _vp, _vp, _vp, _vp], _i),
    "rsp_mask_small_regions_bits": ([_vp, _vp, _i, _i, _i, _i, ctypes.c_longlong, _i, _vp, _vp, _vp, _vp], _i),
    "rsp_panoptic_postprocess": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp,
                                  _vp], _i),
    "rsp_panoptic_postprocess_rescale": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i,
                                          _vp, _vp, _vp, _vp, _vp, _vp], _i),
}


def declared_symbols() -> list[str]:
    """Entry points this binding expects (kept in sync with include/rsp_b200.h by a test)."""
    return sorted(_SIGNATURES)


for _name, (_args, _ret) in _SIGNATURES.items():
    _fn = getattr(_lib, _name)  # AttributeError here = the .so is stale: rebuild
    _fn.argtypes = _args
    _fn.restype = _ret

ABI_VERSION = _lib.rsp_abi_version()

# number of kernel launches issued through this binding (bench.py reports it)
launch_count = 0

# optional launch log of the tensor-core kernels: when `trace` is a list every GEMM / attention wrapper appends
# dict(kind, scope, flops) in launch order (bench.py maps CUPTI kernel records onto it for the roofline)
trace: list | None = None
trace_scope = ""


def _log(kind: str, flops: float) -> None:
    if trace is not None:
        trace.append(dict(kind=kind, scope=trace_scope, flops=float(flops)))


def _check(status: int, what: str) -> None:
    if status != 0:
        msg = _lib.rsp_last_error()
        raise RspError(f"{what} failed (status {status}): {msg.decode() if msg else ''}")


def _ptr(t: torch.Tensor | None) -> int | None:
    if t is None:
        return None
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _require_cuda(*ts: torch.Tensor | None) -> None:
    cur = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RspError("rsprompter_b200 kernels take CUDA tensors only (there is no CPU path)")
        if cur is None:
            cur = torch.cuda.current_device()
        if t.device.index != cur:   # launches go to the current device's current stream
            raise RspError(f"tensor on cuda:{t.device.index} but the current device is cuda:{cur}: "
                           "wrap the call in torch.cuda.device(...) (one process per GPU is the supported layout)")


def _host_f4(v):
    """4 floats as a host C array (DeltaXYWHBBoxCoder target_stds and similar by-value parameters)."""
    v = tuple(float(x) for x in v)
    assert len(v) == 4
    return (ctypes.c_float * 4)(*v)


ACT = {None: 0, "none": 0, "gelu": 1, "relu": 2}


def gemm(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, *,
         out: torch.Tensor | None = None, out_dtype: torch.dtype = torch.bfloat16,
         act: str | None = None, residual: torch.Tensor | None = None, res_mod: int = 0,
         row_map: torch.Tensor | None = None, out_rows: int | None = None,
         simt: bool = False, ln: tuple | None = None, ln64_gelu: tuple | None = None,
         res_block_map: torch.Tensor | None = None, res_block_rows: int = 0) -> torch.Tensor:
    """``out[row_map[m]] = act(a @ w.T + bias) + residual`` (see rsp_gemm_bf16 / _ex in the header).

    a: bf16 [M, K] (row stride may exceed K); w: bf16 [N, K]; bias fp32 [N].
    ln=(gamma, beta, eps): LayerNorm over the whole output row after bias + residual (N <= 256).
    ln64_gelu=(gamma, beta, eps): LayerNorm over each 64-column group, then GELU (bf16 out)."""
    global launch_count
    _require_cuda(a, w, bias, out, residual, row_map, res_block_map)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16, "gemm operands must be bf16"
    assert a.dim() == 2 and w.dim() == 2 and a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N, K2 = w.shape
    assert K == K2, f"gemm K mismatch {K} vs {K2}"
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N and bias.is_contiguous()
    if out is None:
        rows = out_rows if out_rows is not None else M
        out = torch.empty((rows, N), device=a.device, dtype=out_dtype)
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape[1] >= N
    assert out.dtype in (torch.bfloat16, torch.float32)
    ldr = 0
    res_fp32 = 1
    if residual is not None:
        assert residual.dim() == 2 and residual.stride(1) == 1
        assert residual.dtype in (torch.bfloat16, torch.float32)
        ldr = residual.stride(0)
        res_fp32 = int(residual.dtype == torch.float32)
    if row_map is not None:
        assert row_map.dtype == torch.int32 and row_map.numel() == M and row_map.is_contiguous()
    if res_block_map is not None:
        assert res_block_map.dtype == torch.int32 and res_block_map.is_contiguous() and res_block_rows > 0
    epi, g, b, eps = 0, None, None, 1e-6
    if ln is not None:
        epi, (g, b, eps) = 1, ln
    elif ln64_gelu is not None:
        epi, (g, b, eps) = 2, ln64_gelu
    if epi or res_block_map is not None:
        assert not simt
        if g is not None:
            assert g.dtype == torch.float32 and b.dtype == torch.float32 and g.is_contiguous() and b.is_contiguous()
        st = _lib.rsp_gemm_bf16_ex(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0),
                                   M, N, K, _ptr(bias), _ptr(residual), ldr, res_fp32, res_mod,
                                   _ptr(row_map), ACT[act], int(out.dtype == torch.float32), epi,
                                   _ptr(g), _ptr(b), float(eps), _ptr(res_block_map), res_block_rows,
                                   None, None, 0, 0, _stream())
    else:
        fn = _lib.rsp_gemm_bf16_simt if simt else _lib.rsp_gemm_bf16
        st = fn(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0), M, N, K, _ptr(bias),
                _ptr(residual), ldr, res_fp32, res_mod, _ptr(row_map), ACT[act],
                int(out.dtype == torch.float32), _stream())
    _check(st, "rsp_gemm_bf16")
    launch_count += 1
    if not simt:
        _log("gemm", 2.0 * M * N * K)
    return out


def conv3x3_ok(B: int, H: int, W: int, C: int) -> bool:
    return bool(_lib.rsp_conv3x3_geometry_ok(B, H, W, C))


def conv3x3_nhwc(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, *, act: str | None = None,
                 residual: torch.Tensor | None = None, out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 convolution as an implicit GEMM: x bf16 [B,H,W,C], w bf16 [N, 9*C] (ky, kx, c)
    -> [B*H*W, N] = act(conv + bias) + residual."""
    global launch_count
    _require_cuda(x, w, bias, residual)
    B, H, W, C = x.shape
    N = w.shape[0]
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and w.dtype == torch.bfloat16 and w.stride(1) == 1
    assert w.shape[1] == 9 * C
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N and bias.is_contiguous()
    ldr, res_fp32 = 0, 1
    if residual is not None:
        assert residual.dim() == 2 and residual.stride(1) == 1 and residual.shape[0] == B * H * W
        ldr, res_fp32 = residual.stride(0), int(residual.dtype == torch.float32)
    out = torch.empty(B * H * W, N, device=x.device, dtype=out_dtype)
    _check(_lib.rsp_conv3x3_nhwc_bf16(_ptr(x), B, H, W, C, _ptr(w), w.stride(0), _ptr(out), out.stride(0), N, _ptr(bias),
                                      _ptr(residual), ldr, res_fp32, ACT[act], int(out_dtype == torch.float32),
                                      _stream()), "rsp_conv3x3_nhwc_bf16")
    launch_count += 1
    _log("gemm", 2.0 * B * H * W * N * 9 * C)
    return out


def gemm_upscale_mask(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, hyper: torch.Tensor,
                      grid_h: int, grid_w: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """Second mask upscale + GELU + hypernetwork product in one GEMM (epi_mode 3).

    a: bf16 [P*4*h*w, 64] rows (prompt, y, x, tap1); w: bf16 [128, 64] rows (tap2, 32 ch);
    hyper fp32 [P, 32] -> fp32 masks [P, 4h, 4w]."""
    global launch_count
    _require_cuda(a, w, bias, hyper, out)
    M, K = a.shape
    P = M // (4 * grid_h * grid_w)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and w.shape == (128, K)
    assert hyper.dtype == torch.float32 and hyper.shape == (P, 32) and hyper.is_contiguous()
    assert bias.dtype == torch.float32 and bias.numel() == 128
    if out is None:
        out = torch.empty((P, 4 * grid_h, 4 * grid_w), device=a.device, dtype=torch.float32)
    assert out.is_contiguous() and out.dtype == torch.float32
    st = _lib.rsp_gemm_bf16_ex(_ptr(a), a.stride(0), _ptr(w), w.stride(0), None, 0, M, 128, K, _ptr(bias),
                               None, 0, 1, 0, None, 0, 0, 3, None, None, 0.0, None, 0, _ptr(hyper),
                               _ptr(out), grid_h, grid_w, _stream())
    _check(st, "rsp_gemm_bf16_ex(upscale_mask)")
    launch_count += 1
    _log("gemm", 2.0 * M * 128 * K)
    return out


def gemm_upscale_masks(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, hyper: torch.Tensor,
                       grid_h: int, grid_w: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """gemm_upscale_mask for n_out <= 3 hypernetwork vectors per prompt in one GEMM (rsp_gemm_upscale_masks).

    a: bf16 [P*4*h*w, 64]; hyper fp32 [P, n_out, 32] -> fp32 masks [P, n_out, 4h, 4w]; mask o equals
    gemm_upscale_mask(a, w, bias, hyper[:, o]) byte for byte."""
    global launch_count
    _require_cuda(a, w, bias, hyper, out)
    M, K = a.shape
    P = M // (4 * grid_h * grid_w)
    assert a.dtype == torch.bfloat16 and a.stride(1) == 1 and w.dtype == torch.bfloat16 and w.shape == (128, K)
    assert hyper.dtype == torch.float32 and hyper.dim() == 3 and hyper.shape[0] == P and hyper.shape[2] == 32
    assert hyper.is_contiguous() and bias.dtype == torch.float32 and bias.numel() == 128 and bias.is_contiguous()
    n_out = hyper.shape[1]
    if out is None:
        out = torch.empty((P, n_out, 4 * grid_h, 4 * grid_w), device=a.device, dtype=torch.float32)
    assert out.is_contiguous() and out.dtype == torch.float32 and out.shape == (P, n_out, 4 * grid_h, 4 * grid_w)
    st = _lib.rsp_gemm_upscale_masks(_ptr(a), a.stride(0), _ptr(w), w.stride(0), M, K, _ptr(bias), _ptr(hyper), n_out,
                                     _ptr(out), grid_h, grid_w, _stream())
    _check(st, "rsp_gemm_upscale_masks")
    launch_count += 1
    _log("gemm", 2.0 * M * 128 * K)
    return out


def sam_mask_embed(masks: torch.Tensor, weights: list, eps: float = 1e-6) -> torch.Tensor:
    """SamMaskEmbedding: masks fp32 [B, 4h, 4w] -> dense fp32 [B*h*w, 256] channels-last rows (rsp_sam_mask_embed).
    weights = 10 fp32 tensors (conv1 w,b, ln1 g,b, conv2 w,b, ln2 g,b, conv3 w,b)."""
    global launch_count
    _require_cuda(masks, *weights)
    B, hm, wm = masks.shape
    assert masks.dtype == torch.float32 and masks.is_contiguous() and len(weights) == 10
    for t in weights:
        assert t.dtype == torch.float32 and t.is_contiguous()
    h, w = hm // 4, wm // 4
    wp = (ctypes.c_void_p * 10)(*[t.data_ptr() for t in weights])
    dense = torch.empty(B * h * w, 256, device=masks.device, dtype=torch.float32)
    _check(_lib.rsp_sam_mask_embed(_ptr(masks), ctypes.cast(wp, _vp), B, hm, wm, h, w, float(eps), _ptr(dense),
                                   _stream()), "rsp_sam_mask_embed")
    launch_count += 1
    return dense


def add_cast_bf16(a: torch.Tensor, b: torch.Tensor | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
    """bf16(a + b) for fp32 a; b is broadcast over leading dims when smaller (numel divides)."""
    global launch_count
    _require_cuda(a, b, out)
    assert a.dtype == torch.float32 and a.is_contiguous()
    b_mod = 0
    if b is not None:
        assert b.dtype == torch.float32 and b.is_contiguous() and a.numel() % b.numel() == 0
        b_mod = b.numel() if b.numel() != a.numel() else 0
    if out is None:
        out = torch.empty(a.shape, device=a.device, dtype=torch.bfloat16)
    _check(_lib.rsp_add_cast_bf16(_ptr(a), _ptr(b), _ptr(out), a.numel(), b_mod, _stream()), "rsp_add_cast_bf16")
    launch_count += 1
    return out


def token_self_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """q, k, v bf16 [N, T, heads*c] -> bf16 [N, T, heads*c]."""
    global launch_count
    _require_cuda(q, k, v)
    N, T, D = q.shape
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.is_contiguous() and t.shape == (N, T, D)
    out = torch.empty_like(q)
    _check(_lib.rsp_token_self_attention(_ptr(q), _ptr(k), _ptr(v), _ptr(out), N, T, heads, D // heads, _stream()),
           "rsp_token_self_attention")
    launch_count += 1
    return out


def t2i_attention(q: torch.Tensor, K: torch.Tensor, V: torch.Tensor, hw: int,
                  kv_block: torch.Tensor | None = None) -> torch.Tensor:
    """q bf16 [N, Tq, 128]; K, V bf16 [blocks*hw, 128] (row views with a common stride, e.g. the two halves of a
    fused k|v projection); kv_block int32 [N] -> bf16 [N, Tq, 128]."""
    global launch_count
    _require_cuda(q, K, V, kv_block)
    N, Tq, C = q.shape
    assert C == 128 and q.dtype == torch.bfloat16 and q.is_contiguous()
    assert K.dtype == torch.bfloat16 and V.dtype == torch.bfloat16 and K.stride(1) == 1 and V.stride(1) == 1
    assert K.stride(0) == V.stride(0)
    assert K.shape[1] == 128 and V.shape == K.shape and K.shape[0] % hw == 0
    if kv_block is not None:
        assert kv_block.dtype == torch.int32 and kv_block.numel() == N and kv_block.is_contiguous()
    else:
        assert K.shape[0] == N * hw
    out = torch.empty_like(q)
    _check(_lib.rsp_t2i_attention(_ptr(q), _ptr(K), _ptr(V), K.stride(0), _ptr(kv_block), _ptr(out), N, Tq, hw, _stream()),
           "rsp_t2i_attention")
    launch_count += 1
    return out


def t2i_fused(q: torch.Tensor, keys: torch.Tensor, kvw: torch.Tensor, kvb: torch.Tensor, pe_kv: torch.Tensor,
              hw: int) -> torch.Tensor:
    """t2i_attention(q, K, V, hw) with [K | V] = gemm(keys, kvw, kvb, residual=pe_kv, res_mod=hw) computed on chip.

    q bf16 [N, Tq, 128]; keys bf16 [N*hw, 256] (row stride may exceed 256); kvw bf16 [256, 256]; kvb fp32 [256];
    pe_kv bf16 [hw, 256] -> bf16 [N, Tq, 128], the same bytes as the two-call chain."""
    global launch_count
    _require_cuda(q, keys, kvw, kvb, pe_kv)
    N, Tq, C = q.shape
    assert C == 128 and q.dtype == torch.bfloat16 and q.is_contiguous()
    assert keys.dtype == torch.bfloat16 and keys.dim() == 2 and keys.stride(1) == 1 and keys.shape == (N * hw, 256)
    assert kvw.dtype == torch.bfloat16 and kvw.shape == (256, 256) and kvw.is_contiguous()
    assert kvb.dtype == torch.float32 and kvb.numel() == 256 and kvb.is_contiguous()
    assert pe_kv.dtype == torch.bfloat16 and pe_kv.shape == (hw, 256) and pe_kv.is_contiguous()
    out = torch.empty_like(q)
    _check(_lib.rsp_t2i_fused(_ptr(keys), keys.stride(0), _ptr(kvw), _ptr(kvb), _ptr(pe_kv), _ptr(q), _ptr(out), N, Tq,
                              hw, _stream()), "rsp_t2i_fused")
    launch_count += 1
    _log("gemm", 2.0 * N * hw * 256 * 256)
    return out


def i2t_fused(keys: torch.Tensor, wq: torch.Tensor, qb: torch.Tensor, pe_q: torch.Tensor, ktok: torch.Tensor,
              vtok: torch.Tensor, wo: torch.Tensor, ob: torch.Tensor, ln: tuple, hw: int) -> torch.Tensor:
    """LN((i2t(Q, ktok, vtok) @ wo.T + ob) + keys) with Q = gemm(keys, wq, qb, residual=pe_q, res_mod=hw), on chip.

    keys bf16 [N*hw, 256] (row stride may exceed 256; also the residual); wq bf16 [128, 256]; qb fp32 [128];
    pe_q bf16 [hw, 128]; ktok, vtok bf16 [N, Tq, 128]; wo bf16 [256, 128]; ob fp32 [256]; ln = (gamma, beta, eps);
    hw % 64 == 0 -> bf16 [N*hw, 256], the same bytes as the three-call chain."""
    global launch_count
    g, b, eps = ln
    _require_cuda(keys, wq, qb, pe_q, ktok, vtok, wo, ob, g, b)
    N, Tq, C = ktok.shape
    assert C == 128 and hw % 64 == 0
    assert keys.dtype == torch.bfloat16 and keys.dim() == 2 and keys.stride(1) == 1 and keys.shape == (N * hw, 256)
    for t, shape in ((wq, (128, 256)), (pe_q, (hw, 128)), (ktok, (N, Tq, 128)), (vtok, (N, Tq, 128)), (wo, (256, 128))):
        assert t.dtype == torch.bfloat16 and t.shape == shape and t.is_contiguous()
    for t, n in ((qb, 128), (ob, 256), (g, 256), (b, 256)):
        assert t.dtype == torch.float32 and t.numel() == n and t.is_contiguous()
    out = torch.empty((N * hw, 256), device=keys.device, dtype=torch.bfloat16)
    _check(_lib.rsp_i2t_fused(_ptr(keys), keys.stride(0), _ptr(wq), _ptr(qb), _ptr(pe_q), _ptr(ktok), _ptr(vtok),
                              _ptr(wo), _ptr(ob), _ptr(g), _ptr(b), float(eps), _ptr(out), N, Tq, hw, _stream()),
           "rsp_i2t_fused")
    launch_count += 1
    _log("gemm", 2.0 * N * hw * 256 * 256)
    return out


def i2t_attention(Q: torch.Tensor, ktok: torch.Tensor, vtok: torch.Tensor, hw: int,
                  q_block: torch.Tensor | None = None) -> torch.Tensor:
    """Q bf16 [blocks*hw, 128]; ktok, vtok bf16 [N, Tq, 128] -> bf16 [N*hw, 128]."""
    global launch_count
    _require_cuda(Q, ktok, vtok, q_block)
    N, Tq, C = ktok.shape
    assert C == 128 and Q.dtype == torch.bfloat16 and Q.is_contiguous() and Q.shape[1] == 128
    assert ktok.dtype == torch.bfloat16 and vtok.dtype == torch.bfloat16
    assert ktok.is_contiguous() and vtok.is_contiguous() and vtok.shape == ktok.shape
    if q_block is not None:
        assert q_block.dtype == torch.int32 and q_block.numel() == N and q_block.is_contiguous()
    else:
        assert Q.shape[0] == N * hw
    out = torch.empty((N * hw, 128), device=Q.device, dtype=torch.bfloat16)
    _check(_lib.rsp_i2t_attention(_ptr(Q), _ptr(q_block), _ptr(ktok), _ptr(vtok), _ptr(out), N, Tq, hw, _stream()),
           "rsp_i2t_attention")
    launch_count += 1
    return out


def vit_attention(qkv: torch.Tensor, rel_h: torch.Tensor, rel_w: torch.Tensor, n_seq: int, S: int,
                  H: int, hd: int, *, out: torch.Tensor | None = None, simt: bool = False,
                  out_row_map: torch.Tensor | None = None, out_rows: int | None = None) -> torch.Tensor:
    """softmax(q k^T / sqrt(hd) + decomposed rel-pos) v for n_seq sequences of S*S tokens.
    out_row_map (int32 [n_seq*T], -1 = drop) scatters the rows into an [out_rows, D] tensor (window un-partition)."""
    global launch_count
    _require_cuda(qkv, rel_h, rel_w, out)
    T = S * S
    D = H * hd
    if not simt and out_row_map is None and S not in (14, 32, 64) and T % 128 == 0 and S % 4 == 0:
        return vit_attention_generic(qkv, rel_h, rel_w, n_seq, S, H, hd, out=out)
    if not simt and S in (14, 32, 64):     # QK^T + PV on the tensor cores (rel-pos prologue not counted)
        _log("attention_window" if S == 14 else "attention_global", 4.0 * n_seq * H * T * T * hd)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (n_seq * T, 3 * D)
    assert rel_h.dtype == torch.bfloat16 and rel_h.is_contiguous() and rel_h.shape == (2 * S - 1, hd)
    assert rel_w.dtype == torch.bfloat16 and rel_w.is_contiguous() and rel_w.shape == (2 * S - 1, hd)
    if out_row_map is not None:
        assert not simt and out_row_map.dtype == torch.int32 and out_row_map.is_contiguous()
        assert out_row_map.numel() == n_seq * T and out_rows is not None
        _require_cuda(out_row_map)
        if out is None:
            out = torch.empty((out_rows, D), device=qkv.device, dtype=torch.bfloat16)
        assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape == (out_rows, D)
        _check(_lib.rsp_vit_attention_scatter(_ptr(qkv), _ptr(rel_h), _ptr(rel_w), _ptr(out), n_seq, T, S, H, hd,
                                              _ptr(out_row_map), _stream()), "rsp_vit_attention_scatter")
        launch_count += 1
        return out
    if out is None:
        out = torch.empty((n_seq * T, D), device=qkv.device, dtype=torch.bfloat16)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape == (n_seq * T, D)
    fn = _lib.rsp_vit_attention_simt if simt else _lib.rsp_vit_attention
    _check(fn(_ptr(qkv), _ptr(rel_h), _ptr(rel_w), _ptr(out), n_seq, T, S, H, hd, _stream()),
           "rsp_vit_attention")
    launch_count += 1
    return out


def gemm_grouped(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, N: int, m_group_rows: int, w_group_rows: int,
                 row_map: torch.Tensor | None = None) -> torch.Tensor:
    """out[row_map[m], n] = sum_k a[m, k] * w[(m // m_group_rows) * w_group_rows + n, k]: one [N, K] weight per row
    group of a (m_group_rows % 128 == 0).  a bf16 [M, K]; w bf16 [groups * w_group_rows (+ slack), K]."""
    global launch_count
    _require_cuda(a, w, out, row_map)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.dim() == 2 and w.dim() == 2
    assert a.stride(1) == 1 and w.stride(1) == 1 and out.dim() == 2 and out.stride(1) == 1
    M, K = a.shape
    assert w.shape[1] == K and M % m_group_rows == 0 and m_group_rows % 128 == 0
    assert w.shape[0] >= (M // m_group_rows - 1) * w_group_rows + N and out.shape[1] >= N
    assert out.dtype in (torch.bfloat16, torch.float32)
    if row_map is not None:
        assert row_map.dtype == torch.int32 and row_map.numel() == M and row_map.is_contiguous()
    _check(_lib.rsp_gemm_bf16_grouped(_ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(out), out.stride(0), M, N, K,
                                      m_group_rows, w_group_rows, _ptr(row_map), int(out.dtype == torch.float32),
                                      _stream()), "rsp_gemm_bf16_grouped")
    launch_count += 1
    _log("gemm", 2.0 * M * N * K)
    return out


_head_scatter_maps: dict = {}


def vit_attention_generic(qkv: torch.Tensor, rel_h: torch.Tensor, rel_w: torch.Tensor, n_seq: int, S: int, H: int,
                          hd: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """Global attention on any grid with S % 4 == 0 and T % 128 == 0 (S = 48 / 80 for 768^2 / 1280^2 inputs): per
    image, all heads batched along the rows - grouped wgmma GEMMs for Q K^T and P V, one GEMM for Q [Rh; Rw]^T, the
    softmax + decomposed rel-pos row kernel in between.  Intermediates per image: fp32 [H*T, T] scores, bf16 [H*T, T]
    probabilities (2.6 + 1.3 GB for ViT-H at 1280^2), reused across images."""
    global launch_count
    _require_cuda(qkv, rel_h, rel_w, out)
    T, D = S * S, H * hd
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (n_seq * T, 3 * D)
    assert T % 128 == 0 and S % 4 == 0 and hd % 8 == 0, "generic attention path: T % 128 == 0, S % 4 == 0"
    dev = qkv.device
    if out is None:
        out = torch.empty((n_seq * T, D), device=dev, dtype=torch.bfloat16)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape == (n_seq * T, D)
    NT = (2 * S - 1 + 15) // 16 * 16
    tabs = torch.zeros(2 * NT, hd, device=dev, dtype=torch.bfloat16)      # [Rh; Rw], zero rows as padding
    tabs[:2 * S - 1] = rel_h
    tabs[NT:NT + 2 * S - 1] = rel_w
    qh = torch.empty(n_seq, H * T, hd, device=dev, dtype=torch.bfloat16)
    kh = torch.empty(n_seq, H * T, hd, device=dev, dtype=torch.bfloat16)
    vt = torch.empty(n_seq, D, T, device=dev, dtype=torch.bfloat16)
    _check(_lib.rsp_split_heads(_ptr(qkv), 3 * D, 0, H, hd, n_seq, T, _ptr(qh), _stream()), "rsp_split_heads")
    _check(_lib.rsp_split_heads(_ptr(qkv), 3 * D, D, H, hd, n_seq, T, _ptr(kh), _stream()), "rsp_split_heads")
    _check(_lib.rsp_transpose_cols(_ptr(qkv), 3 * D, 2 * D, D, n_seq, T, _ptr(vt), _stream()), "rsp_transpose_cols")
    launch_count += 3
    key = (T, H, dev)
    if key not in _head_scatter_maps:        # stacked row (h, t) -> row t * H + h of the image's [T * H, hd] view
        t = torch.arange(T, device=dev, dtype=torch.int32)
        h = torch.arange(H, device=dev, dtype=torch.int32)
        _head_scatter_maps[key] = (t.view(1, T) * H + h.view(H, 1)).reshape(-1).contiguous()
    rmap = _head_scatter_maps[key]
    scores = torch.empty(H * T, T, device=dev, dtype=torch.float32)
    tab = torch.empty(H * T, 2 * NT, device=dev, dtype=torch.float32)
    P = torch.empty(H * T, T, device=dev, dtype=torch.bfloat16)
    scale = float(hd) ** -0.5
    for b in range(n_seq):
        gemm_grouped(qh[b], kh[b], scores, T, T, T)
        gemm(qh[b], tabs, out=tab)
        _check(_lib.rsp_attn_softmax_bias(_ptr(scores), T, _ptr(tab), 2 * NT, NT, _ptr(P), T, H * T, T, S, scale,
                                          _stream()), "rsp_attn_softmax_bias")
        launch_count += 1
        gemm_grouped(P, vt[b], out[b * T:(b + 1) * T].view(T * H, hd), hd, T, hd, row_map=rmap)
    return out      # (its GEMM launches are in the launch log as kind "gemm")


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, *,
              out: torch.Tensor | None = None, out_dtype: torch.dtype = torch.bfloat16,
              src_map: torch.Tensor | None = None, gelu: bool = False,
              copy_out: torch.Tensor | None = None) -> torch.Tensor:
    """Row LayerNorm of x [rows, C] (fp32 or bf16); optional gather map (-1 -> zero row); copy_out (bf16, same shape
    as x, fp32 x only) also receives a bf16 copy of every source row read."""
    global launch_count
    _require_cuda(x, gamma, beta, out, src_map, copy_out)
    if copy_out is not None:
        assert x.dtype == torch.float32 and copy_out.dtype == torch.bfloat16 and copy_out.shape == x.shape
        assert copy_out.stride(1) == 1
    assert x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.float32, torch.bfloat16)
    C = x.shape[1]
    assert gamma.dtype == torch.float32 and beta.dtype == torch.float32
    assert gamma.numel() == C and beta.numel() == C and gamma.is_contiguous() and beta.is_contiguous()
    rows_out = src_map.numel() if src_map is not None else x.shape[0]
    if src_map is not None:
        assert src_map.dtype == torch.int32 and src_map.is_contiguous()
    if out is None:
        out = torch.empty((rows_out, C), device=x.device, dtype=out_dtype)
    assert out.shape == (rows_out, C) and out.stride(1) == 1
    _check(_lib.rsp_layernorm(_ptr(x), int(x.dtype == torch.float32), x.stride(0), _ptr(out),
                              int(out.dtype == torch.float32), out.stride(0), _ptr(gamma), _ptr(beta),
                              _ptr(src_map), rows_out, C, float(eps), int(gelu), _ptr(copy_out),
                              copy_out.stride(0) if copy_out is not None else 0, _stream()),
           "rsp_layernorm")
    launch_count += 1
    return out


def patchify16(img: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """fp32 NCHW [B,3,H,W] -> bf16 [B*(H/16)*(W/16), 768] patch rows."""
    global launch_count
    _require_cuda(img, out)
    assert img.dtype == torch.float32 and img.is_contiguous() and img.dim() == 4 and img.shape[1] == 3
    B, _, H, W = img.shape
    rows = B * (H // 16) * (W // 16)
    if out is None:
        out = torch.empty((rows, 768), device=img.device, dtype=torch.bfloat16)
    assert out.shape == (rows, 768) and out.is_contiguous() and out.dtype == torch.bfloat16
    _check(_lib.rsp_patchify16(_ptr(img), _ptr(out), B, H, W, _stream()), "rsp_patchify16")
    launch_count += 1
    return out


def im2col_nhwc(x: torch.Tensor, kh: int, kw: int, stride: int, pad: int,
                out: torch.Tensor | None = None) -> torch.Tensor:
    """bf16 NHWC [B,H,W,C] -> [B*Ho*Wo, kh*kw*C] (tap-major, channel-minor)."""
    global launch_count
    _require_cuda(x, out)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
    B, H, W, C = x.shape
    Ho = (H + 2 * pad - kh) // stride + 1
    Wo = (W + 2 * pad - kw) // stride + 1
    if out is None:
        out = torch.empty((B * Ho * Wo, kh * kw * C), device=x.device, dtype=torch.bfloat16)
    assert out.shape == (B * Ho * Wo, kh * kw * C) and out.is_contiguous()
    _check(_lib.rsp_im2col_nhwc(_ptr(x), _ptr(out), B, H, W, C, kh, kw, stride, pad, _stream()),
           "rsp_im2col_nhwc")
    launch_count += 1
    return out


def nhwc_to_nchw(x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """[B, H, W, C] (bf16 or fp32) -> fp32 [B, C, H, W]."""
    global launch_count
    _require_cuda(x, out)
    assert x.is_contiguous() and x.dim() == 4 and x.dtype in (torch.float32, torch.bfloat16)
    B, H, W, C = x.shape
    if out is None:
        out = torch.empty((B, C, H, W), device=x.device, dtype=torch.float32)
    assert out.shape == (B, C, H, W) and out.is_contiguous() and out.dtype == torch.float32
    _check(_lib.rsp_nhwc_to_nchw(_ptr(x), int(x.dtype == torch.float32), _ptr(out), B, H * W, C, _stream()),
           "rsp_nhwc_to_nchw")
    launch_count += 1
    return out


def cast_bf16(x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """fp32 -> bf16 copy (numel % 4 == 0)."""
    global launch_count
    _require_cuda(x, out)
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    assert out.is_contiguous() and out.numel() == x.numel() and out.dtype == torch.bfloat16
    _check(_lib.rsp_cast_f32_bf16(_ptr(x), _ptr(out), x.numel(), _stream()), "rsp_cast_f32_bf16")
    launch_count += 1
    return out


def add_table_bf16(x: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """bf16 x [B, ...] + fp32 table [...] (broadcast over the leading dim) -> bf16."""
    global launch_count
    _require_cuda(x, table)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and table.dtype == torch.float32 and table.is_contiguous()
    assert x.numel() % table.numel() == 0 and table.numel() % 8 == 0
    out = torch.empty_like(x)
    _check(_lib.rsp_add_table_bf16(_ptr(x), _ptr(table), _ptr(out), x.numel(), table.numel(), _stream()),
           "rsp_add_table_bf16")
    launch_count += 1
    return out


# ------------------------------------------------------------------------------ detection ops
def rpn_decode(head_out: torch.Tensor, topk_idx: torch.Tensor, B: int, H: int, W: int, A: int, stride: int,
               base_anchors: torch.Tensor, img_hw: tuple, min_size: float, boxes: torch.Tensor,
               scores: torch.Tensor, out_off: int, stds=(1.0, 1.0, 1.0, 1.0),
               img_shapes: torch.Tensor | None = None) -> None:
    """Decode the K top anchors of one level into boxes[B, n, 4] / scores[B, n] at column out_off.
    img_shapes: device fp32 [B, 2] (h, w) = every image's own img_shape to clip to (default: img_hw for all)."""
    global launch_count
    _require_cuda(head_out, topk_idx, base_anchors, boxes, scores)
    assert head_out.dtype == torch.float32 and head_out.dim() == 2 and head_out.stride(1) == 1
    assert topk_idx.dtype == torch.int64 and topk_idx.is_contiguous() and topk_idx.shape[0] == B
    assert boxes.is_contiguous() and scores.is_contiguous() and boxes.dtype == torch.float32
    K = topk_idx.shape[1]
    if img_shapes is not None:
        _require_cuda(img_shapes)
        assert img_shapes.dtype == torch.float32 and img_shapes.is_contiguous() and img_shapes.shape == (B, 2)
        _check(_lib.rsp_rpn_decode_shapes(_ptr(head_out), head_out.stride(0), _ptr(topk_idx), K, B, H, W, A, stride,
                                          _ptr(base_anchors), _host_f4(stds), _ptr(img_shapes), float(min_size), out_off,
                                          scores.shape[1], _ptr(boxes), _ptr(scores), _stream()), "rsp_rpn_decode_shapes")
        launch_count += 1
        return
    _check(_lib.rsp_rpn_decode(_ptr(head_out), head_out.stride(0), _ptr(topk_idx), K, B, H, W, A, stride,
                               _ptr(base_anchors), _host_f4(stds), float(img_hw[0]), float(img_hw[1]), float(min_size),
                               out_off, scores.shape[1], _ptr(boxes), _ptr(scores), _stream()), "rsp_rpn_decode")
    launch_count += 1


def bbox_cls_decode(cls: torch.Tensor, reg: torch.Tensor, rois: torch.Tensor, roi_valid: torch.Tensor | None,
                    C: int, img_hw: tuple, score_thr: float, stds=(0.1, 0.1, 0.2, 0.2),
                    img_shapes: torch.Tensor | None = None):
    """-> scores fp32 [n*C] (-1 filtered), boxes fp32 [n*C, 4], labels int64 [n*C].
    img_shapes: device fp32 [B, 2] (h, w), indexed by rois[:, 0]: per-image clipping (default: img_hw for all)."""
    global launch_count
    _require_cuda(cls, reg, rois, roi_valid)
    n = rois.shape[0]
    assert cls.dtype == torch.float32 and reg.dtype == torch.float32 and rois.dtype == torch.float32
    assert cls.stride(1) == 1 and reg.stride(1) == 1 and rois.is_contiguous() and rois.shape[1] == 5
    scores = torch.empty(n * C, device=cls.device, dtype=torch.float32)
    boxes = torch.empty(n * C, 4, device=cls.device, dtype=torch.float32)
    labels = torch.empty(n * C, device=cls.device, dtype=torch.int64)
    if roi_valid is not None:
        assert roi_valid.dtype == torch.uint8 and roi_valid.numel() == n
    if img_shapes is not None:
        _require_cuda(img_shapes)
        assert img_shapes.dtype == torch.float32 and img_shapes.is_contiguous() and img_shapes.shape[1] == 2
        _check(_lib.rsp_bbox_cls_decode_shapes(_ptr(cls), cls.stride(0), _ptr(reg), reg.stride(0), _ptr(rois),
                                               _ptr(roi_valid), n, C, _host_f4(stds), _ptr(img_shapes), float(score_thr),
                                               _ptr(scores), _ptr(boxes), _ptr(labels), _stream()),
               "rsp_bbox_cls_decode_shapes")
    else:
        _check(_lib.rsp_bbox_cls_decode(_ptr(cls), cls.stride(0), _ptr(reg), reg.stride(0), _ptr(rois),
                                        _ptr(roi_valid), n, C, _host_f4(stds), float(img_hw[0]), float(img_hw[1]),
                                        float(score_thr), _ptr(scores), _ptr(boxes), _ptr(labels), _stream()),
               "rsp_bbox_cls_decode")
    launch_count += 1
    return scores, boxes, labels


def nms_batched(boxes: torch.Tensor, ids: torch.Tensor, nvalid: torch.Tensor, iou_thr: float,
                max_keep: int = 0) -> torch.Tensor:
    """boxes fp32 [B, n, 4] sorted by descending score, ids int64 [B, n], nvalid int32 [B] -> keep uint8 [B, n].
    max_keep > 0: the caller takes only the first max_keep kept candidates; the scan stops once they exist."""
    global launch_count
    _require_cuda(boxes, ids, nvalid)
    B, n, _ = boxes.shape
    assert boxes.dtype == torch.float32 and boxes.is_contiguous()
    assert ids.dtype == torch.int64 and ids.is_contiguous() and ids.shape == (B, n)
    assert nvalid.dtype == torch.int32 and nvalid.numel() == B
    words = (n + 63) // 64
    mask_ws = torch.empty(B * n * words, device=boxes.device, dtype=torch.int64)
    mx = torch.empty(B, device=boxes.device, dtype=torch.float32)
    keep = torch.empty(B, n, device=boxes.device, dtype=torch.uint8)
    _check(_lib.rsp_nms_batched_topk(_ptr(boxes), _ptr(ids), _ptr(nvalid), B, n, float(iou_thr), _ptr(mask_ws),
                                     _ptr(mx), _ptr(keep), int(max_keep), _stream()), "rsp_nms_batched_topk")
    launch_count += 3
    return keep


def compact_keep(keep: torch.Tensor, boxes: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor | None,
                 K: int):
    """-> boxes [B, K, 4], scores [B, K], labels [B, K] | None, index int32 [B, K], counts int32 [B]."""
    global launch_count
    _require_cuda(keep, boxes, scores, labels)
    B, n = keep.shape
    dev = keep.device
    ob = torch.empty(B, K, 4, device=dev, dtype=torch.float32)
    os_ = torch.empty(B, K, device=dev, dtype=torch.float32)
    ol = torch.empty(B, K, device=dev, dtype=torch.int64) if labels is not None else None
    oi = torch.empty(B, K, device=dev, dtype=torch.int32)
    cnt = torch.empty(B, device=dev, dtype=torch.int32)
    assert boxes.is_contiguous() and scores.is_contiguous() and keep.is_contiguous()
    _check(_lib.rsp_compact_keep(_ptr(keep), _ptr(boxes), _ptr(scores), _ptr(labels), B, n, K, _ptr(ob),
                                 _ptr(os_), _ptr(ol), _ptr(oi), _ptr(cnt), _stream()), "rsp_compact_keep")
    launch_count += 1
    return ob, os_, ol, oi, cnt


SOFT_NMS_METHODS = {"naive": 0, "linear": 1, "gaussian": 2}   # mmcv soft_nms method_dict


def soft_nms_workspace_bytes(B: int, n: int, G: int) -> int:
    """Device workspace of soft_nms_batched for B images of n candidates in G id groups (O(B * n))."""
    out = ctypes.c_size_t(0)
    _check(_lib.rsp_soft_nms_workspace_bytes(int(B), int(n), int(G), ctypes.addressof(out)),
           "rsp_soft_nms_workspace_bytes")
    return int(out.value)


def soft_nms_batched(boxes: torch.Tensor, scores: torch.Tensor, ids: torch.Tensor, nvalid: torch.Tensor,
                     num_groups: int, iou_thr: float, sigma: float = 0.5, min_score: float = 1e-3,
                     method: str = "linear", K: int = 0, split_thr: int = 10000):
    """mmcv batched_nms(..., dict(type='soft_nms', ...)) per image on candidates in input order (see
    rsp_soft_nms_batched).  boxes fp32 [B, n, 4], scores fp32 [B, n], ids int64 [B, n] in [0, num_groups), nvalid
    int32 [B] (valid prefix).  K > 0: the first K selections (the loop stops there); K = 0: all n.
    -> boxes [B, K, 4], decayed scores [B, K], labels = ids [B, K], input index int32 [B, K], counts int32 [B]."""
    global launch_count
    _require_cuda(boxes, scores, ids, nvalid)
    B, n, _ = boxes.shape
    assert boxes.dtype == torch.float32 and boxes.is_contiguous()
    assert scores.dtype == torch.float32 and scores.is_contiguous() and scores.shape == (B, n)
    assert ids.dtype == torch.int64 and ids.is_contiguous() and ids.shape == (B, n)
    assert nvalid.dtype == torch.int32 and nvalid.is_contiguous() and nvalid.numel() == B
    if method not in SOFT_NMS_METHODS:
        raise ValueError(f"soft_nms method must be one of {sorted(SOFT_NMS_METHODS)}, got {method!r}")
    K = int(K) if K > 0 else n
    dev = boxes.device
    nbytes = soft_nms_workspace_bytes(B, n, num_groups)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    ob = torch.empty(B, K, 4, device=dev, dtype=torch.float32)
    os_ = torch.empty(B, K, device=dev, dtype=torch.float32)
    ol = torch.empty(B, K, device=dev, dtype=torch.int64)
    oi = torch.empty(B, K, device=dev, dtype=torch.int32)
    cnt = torch.empty(B, device=dev, dtype=torch.int32)
    _check(_lib.rsp_soft_nms_batched(_ptr(boxes), _ptr(scores), _ptr(ids), _ptr(nvalid), B, n, int(num_groups),
                                     float(iou_thr), float(sigma), float(min_score), SOFT_NMS_METHODS[method],
                                     int(split_thr), K, _ptr(ws), nbytes, _ptr(ob), _ptr(os_), _ptr(ol), _ptr(oi),
                                     _ptr(cnt), _stream()), "rsp_soft_nms_batched")
    launch_count += 3
    return ob, os_, ol, oi, cnt


def roi_align_nhwc(feats: list, rois: torch.Tensor, P: int, strides: list, pes: list | None = None,
                   finest_scale: float = 56.0) -> torch.Tensor:
    """feats: bf16 NHWC levels; rois fp32 [n, 5] -> bf16 [n, P*P*C] in (ph, pw, c) order."""
    global launch_count
    _require_cuda(rois, *feats)
    L = len(feats)
    C = feats[0].shape[3]
    n = rois.shape[0]
    for f in feats:
        assert f.dtype == torch.bfloat16 and f.is_contiguous() and f.shape[3] == C
    assert rois.dtype == torch.float32 and rois.is_contiguous() and rois.shape[1] == 5
    fp = (ctypes.c_void_p * L)(*[f.data_ptr() for f in feats])
    pp = None
    if pes is not None:
        for pe, f in zip(pes, feats):
            assert pe.dtype == torch.float32 and pe.is_contiguous() and pe.shape == f.shape[1:]
        pp = (ctypes.c_void_p * L)(*[pe.data_ptr() for pe in pes])
    hs = (ctypes.c_int32 * L)(*[f.shape[1] for f in feats])
    ws = (ctypes.c_int32 * L)(*[f.shape[2] for f in feats])
    sc = (ctypes.c_float * L)(*[1.0 / s for s in strides])
    out = torch.empty(n, P * P * C, device=rois.device, dtype=torch.bfloat16)
    _check(_lib.rsp_roi_align_nhwc(ctypes.cast(fp, _vp), ctypes.cast(pp, _vp) if pp is not None else None,
                                   ctypes.cast(hs, _vp), ctypes.cast(ws, _vp), ctypes.cast(sc, _vp), L,
                                   _ptr(rois), n, C, P, float(finest_scale), _ptr(out), _stream()),
           "rsp_roi_align_nhwc")
    launch_count += 1
    return out


def mask_paste(logits: torch.Tensor, thr: float, *, raw: bool, size: tuple | None = None,
               rescale: tuple | None = None, bits: torch.Tensor | None = None) -> torch.Tensor:
    """Mask logits fp32 [n, hm, wm], resized bilinearly and thresholded: raw=False sigmoid, then >= thr (M:1763-1777);
    raw=True > thr on the resized logits (SAMDet, M:1133-1152).  size = (H, W): one resize; rescale = (batch_hw,
    crop_hw, ori_hw) for a resized / padded image: to batch_hw -> crop -> to ori_hw.  -> bool [n, H, W], or with
    ``bits`` the masks bit-packed into it: record slots uint8 [n, Hr, Wr/8] (Wr % 16 == 0, the mask at each slot's
    top-left, 0 elsewhere) with rescale, uint8 [n, 4hm, 4wm/8] (the x4 resize) without."""
    global launch_count
    _require_cuda(logits, bits)
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.dim() == 3
    assert size is None or rescale is None
    n, hm, wm = logits.shape
    if rescale is not None:
        assert n > 0
        (Hb, Wb), (ch, cw), (H, W) = rescale
    if bits is None:
        out = torch.empty(n, *(size if rescale is None else (H, W)), device=logits.device, dtype=torch.uint8)
    elif rescale is None:
        assert size is None or tuple(size) == (4 * hm, 4 * wm)
        assert bits.dtype == torch.uint8 and bits.is_contiguous() and bits.numel() == n * 4 * hm * (wm // 2)
    else:
        assert bits.dtype == torch.uint8 and bits.is_contiguous() and bits.dim() == 3 and bits.shape[0] == n
    if n == 0:
        return out.view(torch.bool) if bits is None else bits
    mode = 1 if raw else 2
    if not raw and rescale is None and bits is None and logits.numel() % 4:
        mode = 0   # rsp_sigmoid_f32 takes numel % 4 == 0; rsp_mask_paste's mode 0 activates the taps instead
    elif not raw:
        logits = sigmoid_f32(logits)   # activate once per low-res pixel, then paste
    if rescale is None and bits is None:
        _check(_lib.rsp_mask_paste(_ptr(logits), _ptr(out), n, hm, wm, size[0], size[1], float(thr), mode, _stream()),
               "rsp_mask_paste")
    elif rescale is None:
        _check(_lib.rsp_mask_paste_bits(_ptr(logits), _ptr(bits), n, hm, wm, float(thr), mode, _stream()),
               "rsp_mask_paste_bits")
    elif bits is None:
        _check(_lib.rsp_mask_paste_rescale(_ptr(logits), _ptr(out), n, hm, wm, Hb, Wb, ch, cw, H, W, float(thr), mode,
                                           _stream()), "rsp_mask_paste_rescale")
    else:
        _check(_lib.rsp_mask_paste_rescale_bits(_ptr(logits), _ptr(bits), n, hm, wm, Hb, Wb, ch, cw, H, W, bits.shape[1],
                                                bits.shape[2] * 8, float(thr), mode, _stream()),
               "rsp_mask_paste_rescale_bits")
    launch_count += 1
    return out.view(torch.bool) if bits is None else bits


def sam_mask_stats(logits: torch.Tensor, rescale: tuple, mask_threshold: float = 0.0,
                   stability_score_offset: float = 1.0, iou: torch.Tensor | None = None, pred_iou_thresh: float = 0.0,
                   stability_score_thresh: float = 0.0, crop: tuple | None = None):
    """Per-candidate statistics of SAM mask generation (rsp_sam_mask_stats): logits fp32 [n, hm, wm], rescale =
    (pad_hw, reshaped_hw, original_hw) as mask_paste's.  -> counts int32 [n, 3] (> thr + offset, > thr - offset,
    > thr), boxes int32 [n, 4] (HF's inclusive xyxy of > thr), stability fp32 [n], keep bool [n] (None without iou).
    ``crop`` = ((x0, y0, x1, y1), (scene_h, scene_w)): the masks are that crop box of a larger scene, and the keep flag
    also applies HF's crop-edge rule (rsp_sam_mask_stats_crop; needs iou)."""
    global launch_count
    _require_cuda(logits, iou)
    assert crop is None or iou is not None, "the crop-edge rule is part of the keep flag: pass iou"
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.dim() == 3
    n, hm, wm = logits.shape
    (Hb, Wb), (ch, cw), (H, W) = rescale
    dev = logits.device
    counts = torch.empty(n, 3, device=dev, dtype=torch.int32)
    boxes = torch.empty(n, 4, device=dev, dtype=torch.int32)
    stability = torch.empty(n, device=dev, dtype=torch.float32)
    keep = None
    if iou is not None:
        assert iou.dtype == torch.float32 and iou.is_contiguous() and iou.numel() == n
        keep = torch.empty(n, device=dev, dtype=torch.uint8)
    if n == 0:
        return counts, boxes, stability, None if keep is None else keep.view(torch.bool)
    part = torch.empty(n, (H + 15) // 16, 7, device=dev, dtype=torch.int32)
    thr = float(mask_threshold)
    thr_hi, thr_lo = thr + float(stability_score_offset), thr - float(stability_score_offset)
    if crop is None:
        _check(_lib.rsp_sam_mask_stats(_ptr(logits), n, hm, wm, Hb, Wb, ch, cw, H, W, thr, thr_hi, thr_lo, _ptr(iou),
                                       float(pred_iou_thresh), float(stability_score_thresh), _ptr(part), _ptr(counts),
                                       _ptr(boxes), _ptr(stability), _ptr(keep), _stream()), "rsp_sam_mask_stats")
    else:
        (x0, y0, x1, y1), (sh, sw) = crop
        _check(_lib.rsp_sam_mask_stats_crop(_ptr(logits), n, hm, wm, Hb, Wb, ch, cw, H, W, thr, thr_hi, thr_lo,
                                            _ptr(iou), float(pred_iou_thresh), float(stability_score_thresh), int(x0),
                                            int(y0), int(x1), int(y1), int(sh), int(sw), _ptr(part), _ptr(counts),
                                            _ptr(boxes), _ptr(stability), _ptr(keep), _stream()),
               "rsp_sam_mask_stats_crop")
    launch_count += 2
    return counts, boxes, stability, None if keep is None else keep.view(torch.bool)


SMALL_REGION_MODES = {"holes": 0, "islands": 1}     # segment_anything remove_small_regions' modes


def small_regions_ws_bytes(n: int, H: int, W: int) -> int:
    """Device workspace of mask_small_regions_bits for n masks of H x W: 32 bytes per mask and an int32 label per
    2 x 2 pixel block."""
    return n * (32 + 4 * ((H + 1) // 2) * ((W + 1) // 2))


def mask_small_regions_bits(bits: torch.Tensor, W: int, min_area: int, mode: str, out: torch.Tensor | None = None,
                            ws: torch.Tensor | None = None):
    """SAM's remove_small_regions (rsp_mask_small_regions_bits) on bit-packed masks uint8 [n, H, ld] of width W:
    components of the working mask (~mask for mode "holes", mask for "islands") with area < min_area (an int) are
    filled / removed.  -> out uint8 [n, H, ld] (bits at x >= W zero), changed bool [n], boxes int32 [n, 4] (inclusive
    xyxy of out, zeros when empty).  ws: uint8 of at least small_regions_ws_bytes(n, H, W) bytes, or None."""
    global launch_count
    _require_cuda(bits, out, ws)
    assert bits.dtype == torch.uint8 and bits.is_contiguous() and bits.dim() == 3
    n, H, ld = bits.shape
    dev = bits.device
    if out is None:
        out = torch.empty_like(bits)
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.shape == bits.shape
    changed = torch.empty(n, device=dev, dtype=torch.uint8)
    boxes = torch.empty(n, 4, device=dev, dtype=torch.int32)
    if n == 0:
        return out, changed.view(torch.bool), boxes
    if not -2 ** 63 <= int(min_area) < 2 ** 63:
        raise ValueError(f"min_area {min_area} does not fit the kernel's 64-bit threshold")
    need = small_regions_ws_bytes(n, H, W)
    if ws is None:
        ws = torch.empty(need, device=dev, dtype=torch.uint8)
    assert ws.dtype == torch.uint8 and ws.is_contiguous() and ws.numel() >= need
    _check(_lib.rsp_mask_small_regions_bits(_ptr(bits), _ptr(out), n, H, int(W), ld, int(min_area),
                                            SMALL_REGION_MODES[mode], _ptr(ws), _ptr(changed), _ptr(boxes),
                                            _stream()), "rsp_mask_small_regions_bits")
    launch_count += 7
    return out, changed.view(torch.bool), boxes


def sigmoid_f32(x: torch.Tensor) -> torch.Tensor:
    """fp32 sigmoid (numel % 4 == 0), the activation FCNMaskHead / the paste kernels apply once per low-res pixel."""
    global launch_count
    _require_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.numel() % 4 == 0
    out = torch.empty_like(x)
    if x.numel():
        _check(_lib.rsp_sigmoid_f32(_ptr(x), _ptr(out), x.numel(), _stream()), "rsp_sigmoid_f32")
        launch_count += 1
    return out


def mask_paste_boxes(probs: torch.Tensor, boxes: torch.Tensor, size: tuple, thr: float,
                     bits: torch.Tensor | None = None) -> torch.Tensor:
    """FCNMaskHead paste (fcn_mask_head.py:_do_paste_mask + :388-392): probs fp32 [n, hm, wm] sampled into boxes fp32
    [n, 4] on a size = (H, W) canvas, >= thr -> bool [n, H, W]; with ``bits`` (uint8, n * H * W/8 bytes) the result is
    written bit-packed into it (result-record layout) instead."""
    global launch_count
    _require_cuda(probs)
    n, hm, wm = probs.shape
    assert probs.dtype == torch.float32 and probs.is_contiguous() and boxes.dtype == torch.float32
    assert boxes.is_contiguous() and boxes.shape == (n, 4)
    if bits is not None:
        assert bits.dtype == torch.uint8 and bits.is_contiguous() and size[1] % 16 == 0
        assert bits.numel() == n * size[0] * size[1] // 8
        out = bits
    else:
        out = torch.empty(n, size[0], size[1], device=probs.device, dtype=torch.uint8)
    if n > 0:
        _check(_lib.rsp_mask_paste_boxes(_ptr(probs), _ptr(boxes), _ptr(out), n, hm, wm, size[0], size[1], float(thr),
                                         0 if bits is None else 1, _stream()), "rsp_mask_paste_boxes")
        launch_count += 1
    return out if bits is not None else out.view(torch.bool)


def zero_border_nhwc(x: torch.Tensor) -> torch.Tensor:
    """Zero the 1-pixel border of bf16 NHWC maps [N, H, W, C] in place."""
    global launch_count
    _require_cuda(x)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4 and x.shape[3] % 8 == 0
    N, H, W, C = x.shape
    _check(_lib.rsp_zero_border_nhwc(_ptr(x), N, H, W, C, _stream()), "rsp_zero_border_nhwc")
    launch_count += 1
    return x


def pool2_nhwc(x: torch.Tensor, mode: int) -> torch.Tensor:
    """bf16 NHWC: mode 0 = 2x2 max pool stride 2, mode 1 = stride-2 subsample."""
    global launch_count
    _require_cuda(x)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
    B, H, W, C = x.shape
    Ho, Wo = (H // 2, W // 2) if mode == 0 else ((H + 1) // 2, (W + 1) // 2)
    out = torch.empty(B, Ho, Wo, C, device=x.device, dtype=torch.bfloat16)
    _check(_lib.rsp_pool2_nhwc(_ptr(x), _ptr(out), B, H, W, C, mode, _stream()), "rsp_pool2_nhwc")
    launch_count += 1
    return out


def sin_fold(x: torch.Tensor) -> torch.Tensor:
    """fp32 [..., 2k] -> fp32 [..., k]: sin(even) + odd."""
    global launch_count
    _require_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[-1] % 2 == 0
    out = torch.empty(*x.shape[:-1], x.shape[-1] // 2, device=x.device, dtype=torch.float32)
    _check(_lib.rsp_sin_fold(_ptr(x), _ptr(out), out.numel(), _stream()), "rsp_sin_fold")
    launch_count += 1
    return out


def layernorm_add(x: torch.Tensor, residual: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
                  res_block_map: torch.Tensor | None = None, res_block_rows: int = 0,
                  pos: torch.Tensor | None = None):
    """bf16 LayerNorm(x + residual) for bf16 x [rows, C <= 256]; residual fp32 / bf16, optionally block-mapped.
    With pos (fp32 [P, C]) also returns bf16(out + pos[row % P])."""
    global launch_count
    _require_cuda(x, residual, gamma, beta, res_block_map)
    rows, C = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous()
    assert residual.is_contiguous() and residual.shape[1] == C and residual.dtype in (torch.float32, torch.bfloat16)
    assert gamma.dtype == torch.float32 and beta.dtype == torch.float32 and gamma.numel() == C
    if res_block_map is not None:
        assert res_block_map.dtype == torch.int32 and res_block_map.is_contiguous() and res_block_rows > 0
    else:
        assert residual.shape[0] == rows
    out = torch.empty_like(x)
    out_pe, pos_mod = None, 0
    if pos is not None:
        assert pos.dtype == torch.float32 and pos.is_contiguous() and pos.shape[1] == C
        out_pe, pos_mod = torch.empty_like(x), pos.shape[0]
    _check(_lib.rsp_layernorm_add(_ptr(x), _ptr(residual), int(residual.dtype == torch.float32), _ptr(res_block_map),
                                  res_block_rows, _ptr(gamma), _ptr(beta), _ptr(out), _ptr(pos), pos_mod,
                                  _ptr(out_pe), rows, C, float(eps), _stream()), "rsp_layernorm_add")
    launch_count += 1
    return out if pos is None else (out, out_pe)


# ------------------------------------------------------------------------------ query-head ops
def groupnorm_nhwc(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int = 32, eps: float = 1e-5,
                   up: torch.Tensor | None = None, relu: bool = False) -> torch.Tensor:
    """GroupNorm on bf16 NHWC (+ bilinear x2 of `up` added after the affine, + ReLU)."""
    global launch_count
    _require_cuda(x, gamma, beta, up)
    B, H, W, C = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and gamma.dtype == torch.float32 and beta.dtype == torch.float32
    if up is not None:
        assert up.dtype == torch.bfloat16 and up.is_contiguous() and up.shape == (B, H // 2, W // 2, C)
    stats = torch.empty(B * groups * 2 * (1 + (H * W + 255) // 256), device=x.device, dtype=torch.float32)
    out = torch.empty_like(x)
    _check(_lib.rsp_groupnorm_nhwc(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(up), _ptr(out), B, H, W, C,
                                   groups, float(eps), int(relu), _stream()), "rsp_groupnorm_nhwc")
    launch_count += 3
    return out


def ms_deform_attn_sample(value: torch.Tensor, ow: torch.Tensor, shapes: list, points: int) -> torch.Tensor:
    """value bf16 [B, NQ, E] (E = 8 heads x 16 or x 32); ow fp32 [B*NQ, >= 8*L*P*3]; shapes [(h, w)] low -> high res
    -> bf16 [B*NQ, E]."""
    global launch_count
    _require_cuda(value, ow)
    B, NQ, E = value.shape
    L = len(shapes)
    assert E in (128, 256) and value.dtype == torch.bfloat16 and value.is_contiguous()
    assert ow.dtype == torch.float32 and ow.stride(1) == 1 and ow.shape[0] == B * NQ and ow.shape[1] >= 8 * L * points * 3
    hs = (ctypes.c_int32 * L)(*[s[0] for s in shapes])
    ws = (ctypes.c_int32 * L)(*[s[1] for s in shapes])
    out = torch.empty(B * NQ, E, device=value.device, dtype=torch.bfloat16)
    _check(_lib.rsp_ms_deform_attn_sample_c(_ptr(value), _ptr(ow), ow.stride(0), ctypes.cast(hs, _vp), ctypes.cast(ws, _vp),
                                            L, points, B, NQ, _ptr(out), E, _stream()), "rsp_ms_deform_attn_sample_c")
    launch_count += 1
    return out


def mha_small(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, B: int, nq: int, nk: int,
              mask: torch.Tensor | None = None, head_dim: int = 16) -> torch.Tensor:
    """q [B*nq, >=E], k / v [B*nk, >=E] bf16 row views (row stride = leading dim), E = 8 * head_dim (16 or 32);
    mask = bit words int64 [B*nq, ceil(nk/64)] from attn_mask_bits -> bf16 [B*nq, E]."""
    global launch_count
    _require_cuda(q, k, v, mask)
    for t in (q, k, v):
        assert t.dtype == torch.bfloat16 and t.stride(1) == 1
    if mask is not None:
        assert mask.dtype == torch.int64 and mask.is_contiguous() and mask.shape == (B * nq, (nk + 63) // 64)
    assert head_dim in (16, 32)
    out = torch.empty(B * nq, 8 * head_dim, device=q.device, dtype=torch.bfloat16)
    _check(_lib.rsp_mha_small_hd(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(mask), B, nq, nk,
                                 _ptr(out), head_dim, _stream()), "rsp_mha_small_hd")
    launch_count += 1
    return out


def attn_mask_bits(logits: torch.Tensor) -> torch.Tensor:
    """fp32 [rows, nk] level-sized mask logits -> int64 bit words [rows, ceil(nk/64)] (bit set = masked)."""
    global launch_count
    _require_cuda(logits)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    rows, nk = logits.shape
    out = torch.empty(rows, (nk + 63) // 64, device=logits.device, dtype=torch.int64)
    _check(_lib.rsp_attn_mask_bits(_ptr(logits), logits.stride(0), rows, nk, _ptr(out), _stream()), "rsp_attn_mask_bits")
    launch_count += 1
    return out


def resize_bilinear_nhwc(x: torch.Tensor, hw: tuple) -> torch.Tensor:
    """bf16 [B, H, W, C] -> bf16 [B, h, w, C] (F.interpolate bilinear, align_corners=False)."""
    global launch_count
    _require_cuda(x)
    B, H, W, C = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and C % 8 == 0
    out = torch.empty(B, hw[0], hw[1], C, device=x.device, dtype=torch.bfloat16)
    _check(_lib.rsp_resize_bilinear_nhwc(_ptr(x), B, H, W, C, hw[0], hw[1], _ptr(out), _stream()),
           "rsp_resize_bilinear_nhwc")
    launch_count += 1
    return out


def mask_embed_src(mpp: torch.Tensor, weights: list, emb_rows: torch.Tensor, pos_rows: torch.Tensor, n_per_img: int,
                   hw: tuple, eps: float = 1e-6, want_pe: bool = False):
    """-> (src, src_pe) bf16 [N*h*w, 256]; weights = 10 fp32 tensors (conv1 w,b, ln1 g,b, conv2 w,b, ln2 g,b, conv3 w,b)."""
    global launch_count
    _require_cuda(mpp, emb_rows, pos_rows, *weights)
    N, hm, wm = mpp.shape
    h, w = hw
    assert mpp.dtype == torch.float32 and mpp.is_contiguous() and len(weights) == 10
    for t in weights:
        assert t.dtype == torch.float32 and t.is_contiguous()
    assert emb_rows.dtype == torch.float32 and emb_rows.is_contiguous() and pos_rows.dtype == torch.float32
    wp = (ctypes.c_void_p * 10)(*[t.data_ptr() for t in weights])
    src = torch.empty(N * h * w, 256, device=mpp.device, dtype=torch.bfloat16)
    src_pe = torch.empty_like(src) if want_pe else None
    _check(_lib.rsp_mask_embed_src(_ptr(mpp), ctypes.cast(wp, _vp), _ptr(emb_rows), _ptr(pos_rows), N, n_per_img, hm, wm,
                                   h, w, float(eps), _ptr(src), _ptr(src_pe), _stream()), "rsp_mask_embed_src")
    launch_count += 1
    return src, src_pe


def query_postprocess(logits: torch.Tensor, sel: torch.Tensor, cls_scores: torch.Tensor, size: tuple | None = None, *,
                      rescale: tuple | None = None, bits: torch.Tensor | None = None, scores: torch.Tensor | None = None,
                      boxes: torch.Tensor | None = None):
    """logits fp32 [n_maps, hm, wm]; sel int32 [n] map of each instance; cls_scores fp32 [n] -> (masks, scores [n],
    boxes [n, 4]) of the selected maps resized bilinearly: size = (H, W), one resize; rescale = (batch_hw, crop_hw,
    out_hw) for a resized / padded image: to batch_hw -> crop -> to out_hw.  masks bool [n, H, W], or with ``bits``
    bit-packed into it: record slots uint8 [n, Hr, Wr/8] (out_hw mask at each slot's top-left) with rescale, uint8
    [n, 4hm, 4wm/8] (the x4 resize) without.  scores / boxes may be views of a result record."""
    global launch_count
    _require_cuda(logits, sel, cls_scores, bits, scores, boxes)
    n = sel.numel()
    _, hm, wm = logits.shape
    assert logits.dtype == torch.float32 and logits.is_contiguous() and sel.dtype == torch.int32 and cls_scores.dtype == torch.float32
    assert size is None or rescale is None
    if rescale is not None:
        (Hb, Wb), (ch, cw), (H, W) = rescale
    elif bits is not None:
        assert size is None or tuple(size) == (4 * hm, 4 * wm)
        H, W = 4 * hm, 4 * wm
    else:
        H, W = size
    Hr = H
    if bits is None:
        masks = torch.empty(n, H, W, device=logits.device, dtype=torch.uint8)
    else:
        assert sel.is_contiguous() and cls_scores.is_contiguous() and cls_scores.numel() == n
        assert bits.dtype == torch.uint8 and bits.is_contiguous()
        if rescale is None:
            assert bits.numel() == n * H * W // 8
        else:
            assert bits.dim() == 3 and bits.shape[0] == n
            Hr = bits.shape[1]
    if scores is None:
        scores = torch.empty(n, device=logits.device, dtype=torch.float32)
    if boxes is None:
        boxes = torch.empty(n, 4, device=logits.device, dtype=torch.float32)
    assert scores.is_contiguous() and boxes.is_contiguous() and scores.numel() == n and boxes.numel() == 4 * n
    part = torch.empty(n * ((Hr + 15) // 16) * 6, device=logits.device, dtype=torch.float32)
    args = (_ptr(logits), _ptr(sel), _ptr(cls_scores), n, hm, wm)
    tail = (_ptr(masks if bits is None else bits), _ptr(part), _ptr(scores), _ptr(boxes), _stream())
    if rescale is None and bits is None:
        _check(_lib.rsp_query_postprocess(*args, H, W, *tail), "rsp_query_postprocess")
    elif rescale is None:
        _check(_lib.rsp_query_postprocess_bits(*args, *tail), "rsp_query_postprocess_bits")
    elif bits is None:
        _check(_lib.rsp_query_postprocess_rescale(*args, Hb, Wb, ch, cw, H, W, *tail), "rsp_query_postprocess_rescale")
    else:
        _check(_lib.rsp_query_postprocess_rescale_bits(*args, Hb, Wb, ch, cw, H, W, Hr, bits.shape[2] * 8, *tail),
               "rsp_query_postprocess_rescale_bits")
    launch_count += 2
    return (masks.view(torch.bool) if bits is None else bits), scores, boxes


PANOPTIC_INSTANCE_OFFSET = 1000      # mmdet.evaluation.functional.INSTANCE_OFFSET


def check_panoptic_bounds(nq: int, num_classes: int) -> None:
    """ValueError unless the panoptic kernels can represent the result: query indices in uint16 (one value left for
    "no kept query"), labels below INSTANCE_OFFSET, and every segment id (label + instance_id * 1000) in int32."""
    if not 0 < nq <= 65535:
        raise ValueError(f"panoptic post-processing takes 1 to 65535 queries per image, got {nq}")
    if not 0 < num_classes < PANOPTIC_INSTANCE_OFFSET:
        raise ValueError(f"panoptic segment ids hold labels below {PANOPTIC_INSTANCE_OFFSET}, got num_classes "
                         f"{num_classes}")
    if nq * PANOPTIC_INSTANCE_OFFSET + num_classes > 2 ** 31 - 1:
        raise ValueError(f"panoptic segment ids of {nq} queries do not fit in int32")


def panoptic_postprocess(logits: torch.Tensor, keep: torch.Tensor, scores: torch.Tensor, labels: torch.Tensor,
                         num_things: int, num_classes: int, iou_thr: float, filter_low_score: bool,
                         size: tuple | None = None, *, rescale: tuple | None = None):
    """MaskFormerFusionHead.panoptic_postprocess (maskformer_fusion_head.py:41-106) of B images on the device, with no
    host read.  logits fp32 [B*nq, hm, wm] low-res mask logits; keep bool [B, nq]; scores fp32 / labels int [B, nq]
    (softmax max and argmax of the class logits); size = (H, W): one bilinear resize; rescale = (batch_hw, crop_hw,
    out_hw): to batch_hw -> crop -> to out_hw (M:652-656 + 679-691).  -> (pan int32 [B, 1, H, W], dict(mask_area,
    original_area, segment_id) int32 [B, nq]: the per-query counts and written ids, 0 / 0 / -1 for queries not kept)."""
    global launch_count
    B, nq = keep.shape
    check_panoptic_bounds(nq, num_classes)
    assert (size is None) != (rescale is None)
    _require_cuda(logits, keep, scores, labels)
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.shape[0] == B * nq
    _, hm, wm = logits.shape
    H, W = size if rescale is None else rescale[2]
    dev = logits.device
    keep = keep.to(torch.uint8).contiguous()
    scores = scores.to(torch.float32).contiguous()
    labels = labels.to(torch.int32).contiguous()
    idx = torch.empty(B, H * W, device=dev, dtype=torch.int16)
    bits = torch.empty(B, (H * W + 31) // 32, device=dev, dtype=torch.int32)
    areas = torch.empty(2, B, nq, device=dev, dtype=torch.int32)
    seg = torch.empty(B, nq, device=dev, dtype=torch.int32)
    pan = torch.empty(B, 1, H, W, device=dev, dtype=torch.int32)
    thr = ctypes.c_double(float(iou_thr))
    head = (_ptr(logits), _ptr(keep), _ptr(scores), _ptr(labels), B, nq, hm, wm)
    tail = (int(num_things), int(num_classes), ctypes.addressof(thr), int(bool(filter_low_score)), _ptr(idx), _ptr(bits),
            _ptr(areas), _ptr(seg), _ptr(pan), _stream())
    if rescale is None:
        _check(_lib.rsp_panoptic_postprocess(*head, H, W, *tail), "rsp_panoptic_postprocess")
    else:
        (Hb, Wb), (ch, cw), _ = rescale
        _check(_lib.rsp_panoptic_postprocess_rescale(*head, Hb, Wb, ch, cw, H, W, *tail),
               "rsp_panoptic_postprocess_rescale")
    launch_count += 3
    return pan, dict(mask_area=areas[0], original_area=areas[1], segment_id=seg)


# ------------------------------------------------------------------------------ result-record payload
def pack_mask_bits(masks: torch.Tensor, bits: torch.Tensor | None = None) -> torch.Tensor:
    """bool / uint8 [..., W] -> uint8 [..., ceil(W/8)], pixel x = bit x % 8 of byte x // 8."""
    global launch_count
    _require_cuda(masks, bits)
    m = masks.view(torch.uint8) if masks.dtype == torch.bool else masks
    assert m.dtype == torch.uint8 and m.is_contiguous()
    W = m.shape[-1]
    rows = m.numel() // W
    if bits is None:
        bits = torch.empty(*m.shape[:-1], (W + 7) // 8, device=m.device, dtype=torch.uint8)
    assert bits.dtype == torch.uint8 and bits.is_contiguous() and bits.numel() == rows * ((W + 7) // 8)
    if rows:
        _check(_lib.rsp_pack_mask_bits(_ptr(m), _ptr(bits), rows, W, _stream()), "rsp_pack_mask_bits")
        launch_count += 1
    return bits


def unpack_mask_bits(bits: torch.Tensor, W: int) -> torch.Tensor:
    """uint8 [..., ceil(W/8)] -> bool [..., W]."""
    global launch_count
    _require_cuda(bits)
    assert bits.dtype == torch.uint8 and bits.is_contiguous() and bits.shape[-1] == (W + 7) // 8
    out = torch.empty(*bits.shape[:-1], W, device=bits.device, dtype=torch.uint8)
    rows = out.numel() // W
    if rows:
        _check(_lib.rsp_unpack_mask_bits(_ptr(bits), _ptr(out), rows, W, _stream()), "rsp_unpack_mask_bits")
        launch_count += 1
    return out.view(torch.bool)


# ------------------------------------------------------------------------------ DetDataPreprocessor
def _host_f3(v):
    v = tuple(float(x) for x in v)
    assert len(v) == 3
    return (ctypes.c_float * 3)(*v)


def preprocess_u8(img: torch.Tensor, out: torch.Tensor, mean, std, swap_rb: bool, pad_value: float) -> torch.Tensor:
    """img uint8 [3, h, w] (any strides, e.g. a permuted HWC array) -> out fp32 [3, H, W] (a slot of the batch tensor)."""
    global launch_count
    _require_cuda(img, out)
    assert img.dtype == torch.uint8 and img.dim() == 3 and img.shape[0] == 3
    assert out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 3 and out.shape[0] == 3
    _, h, w = img.shape
    sc, sy, sx = img.stride()
    _check(_lib.rsp_preprocess_u8(_ptr(img), h, w, sc, sy, sx, _ptr(out), out.shape[1], out.shape[2], _host_f3(mean),
                                  _host_f3(std), int(swap_rb), float(pad_value), _stream()), "rsp_preprocess_u8")
    launch_count += 1
    return out


def resize_pad_u8(imgs: list, sizes: list, out: torch.Tensor, mean, std, swap_rb: bool, pad) -> torch.Tensor:
    """The keep-ratio Resize + Pad + normalisation of a batch in one launch: imgs = uint8 [3, h, w] device views (any
    strides: CHW planes, permuted HWC arrays, tile views of a scene), sizes = (new_h, new_w) per image, out fp32
    [B, 3, Hp, Wp]; pad = 3 raw pad values in input channel order."""
    global launch_count
    _require_cuda(out, *imgs)
    B = len(imgs)
    assert B == len(sizes) == out.shape[0] and B > 0
    assert out.dtype == torch.float32 and out.is_contiguous() and out.dim() == 4 and out.shape[1] == 3
    rows = []
    for t, (nh, nw) in zip(imgs, sizes):
        assert t.dtype == torch.uint8 and t.dim() == 3 and t.shape[0] == 3
        rows.append([t.data_ptr(), *t.stride(), t.shape[1], t.shape[2], int(nh), int(nw)])
    host = torch.tensor(rows, dtype=torch.int64).pin_memory()
    desc = host.to(out.device, non_blocking=True)
    _check(_lib.rsp_resize_pad_u8(_ptr(desc), host.data_ptr(), B, _ptr(out), out.shape[2], out.shape[3],
                                  _host_f3(mean), _host_f3(std), int(swap_rb), _host_f3(pad), _stream()),
           "rsp_resize_pad_u8")
    launch_count += 1
    return out


def patchify16_u8(img: torch.Tensor, mean, std, swap_rb: bool, out: torch.Tensor | None = None) -> torch.Tensor:
    """uint8 [B,3,H,W] (contiguous, or channels-last memory = decoded HWC images) -> bf16 [B*(H/16)*(W/16), 768]
    normalised patch rows (DetDataPreprocessor fused into the patch-embed operand)."""
    global launch_count
    _require_cuda(img, out)
    assert img.dtype == torch.uint8 and img.dim() == 4 and img.shape[1] == 3
    B, _, H, W = img.shape
    if img.is_contiguous():
        hwc = 0
    else:
        assert img.permute(0, 2, 3, 1).is_contiguous(), "uint8 batch must be NCHW-contiguous or channels-last"
        hwc = 1
    rows = B * (H // 16) * (W // 16)
    if out is None:
        out = torch.empty((rows, 768), device=img.device, dtype=torch.bfloat16)
    assert out.shape == (rows, 768) and out.is_contiguous() and out.dtype == torch.bfloat16
    _check(_lib.rsp_patchify16_u8(_ptr(img), hwc, _ptr(out), B, H, W, _host_f3(mean), _host_f3(std), int(swap_rb),
                                  _stream()), "rsp_patchify16_u8")
    launch_count += 1
    return out


# ------------------------------------------------------------------------------ COCO RLE
def mask_rle(groups: list, packed: bool) -> list:
    """pycocotools compressed RLE strings (bytes, one per mask, in order) of every mask in ``groups`` = [(masks, W)]:
    contiguous CUDA tensors [n, H, W] bool / uint8 (packed=False) or uint8 [n, H, ceil(W/8)] bit-packed rows
    (packed=True), sizes free to differ between groups.  One batched encode: a length pass + offset scan, one
    device->host read of the total, the write pass, one copy of the chars + lengths."""
    global launch_count
    groups = [(t, int(W)) for t, W in groups if t.shape[0] > 0]
    if not groups:
        return []
    _require_cuda(*[t for t, _ in groups])
    base = min(t.data_ptr() for t, _ in groups)        # descriptors address every mask from the lowest pointer
    rows = []
    for t, W in groups:
        assert t.dtype in (torch.bool, torch.uint8) and t.dim() == 3 and t.is_contiguous()
        n, H, ld = t.shape
        assert ld == ((W + 7) // 8 if packed else W), "row length does not match W"
        off = t.data_ptr() - base
        rows += [(off + j * H * ld, H, W) for j in range(n)]
    return _rle_strings(base, packed, rows, groups[0][0].device, placed=False)


def mask_rle_placed(groups: list, packed: bool) -> list:
    """pycocotools compressed RLE strings (bytes, in order) of canvases that hold one mask each, the canvas itself never
    formed.  ``groups`` = [(src, placements)], src a contiguous CUDA tensor (bool / uint8 pixels, or bit-packed rows
    with packed=True) and placements = [(byte offset in src, row bytes, rows, h, w, H, W, y0, x0)]: the H x W canvas is
    zero but for canvas[y0:y0 + h, x0:x0 + w] = mask[:h, :w], the mask's rows of ``row bytes`` starting at that offset.
    The work is proportional to h x w; host syncs and copies as mask_rle."""
    groups = [(t, list(pl)) for t, pl in groups if len(pl) > 0]
    if not groups:
        return []
    _require_cuda(*[t for t, _ in groups])
    base = min(t.data_ptr() for t, _ in groups)
    rows = []
    for t, pl in groups:
        assert t.is_contiguous() and t.dtype in (torch.bool, torch.uint8)
        shift = t.data_ptr() - base
        for p in pl:
            off, ld, nrows, h, w, H, W, y0, x0 = (int(v) for v in p)
            # the kernel reads rows [0, h) of the mask, from its offset on
            assert 0 <= off and off + (h - 1) * ld + ((w + 7) // 8 if packed else w) <= t.numel(), "mask outside src"
            rows.append((off + shift, ld, nrows, h, w, H, W, y0, x0))
    return _rle_strings(base, packed, rows, groups[0][0].device, placed=True)


def _rle_strings(base: int, packed: bool, rows: list, dev, placed: bool) -> list:
    """The length pass + offset scan, one device->host read of the total, the write pass, one copy of the chars."""
    global launch_count
    n = len(rows)
    lengths_fn, write_fn = ((_lib.rsp_mask_rle_placed_lengths, _lib.rsp_mask_rle_placed_write) if placed else
                            (_lib.rsp_mask_rle_lengths, _lib.rsp_mask_rle_write))
    what = "rsp_mask_rle_placed" if placed else "rsp_mask_rle"
    desc_host = torch.tensor(rows, dtype=torch.int64).pin_memory()
    desc = desc_host.to(dev, non_blocking=True)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    _check(lengths_fn(base, int(packed), _ptr(desc), _ptr(desc_host), n, _ptr(offsets), _stream()), what + "_lengths")
    total = int(offsets[n].item())                       # host sync 1: the exact pool size
    pool = torch.empty(total, dtype=torch.uint8, device=dev)
    lengths = torch.empty(n, dtype=torch.int32, device=dev)
    _check(write_fn(base, int(packed), _ptr(desc), n, _ptr(offsets), _ptr(pool), _ptr(lengths), _stream()),
           what + "_write")
    launch_count += 3
    host_pool = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    host_len = torch.empty(n, dtype=torch.int32, pin_memory=True)
    host_pool.copy_(pool, non_blocking=True)
    host_len.copy_(lengths, non_blocking=True)
    torch.cuda.current_stream().synchronize()            # host sync 2: chars + lengths
    lens = host_len.tolist()
    if min(lens) < 0:
        raise RspError(what + "_write: a mask's RLE string is longer than 2^31 - 1 chars")
    buf = host_pool.numpy().tobytes()
    out, p = [], 0
    for ln in lens:
        out.append(buf[p:p + ln])
        p += ln
    return out
