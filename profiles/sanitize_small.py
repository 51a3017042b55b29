"""Tiny invocations of the kernels added in round 2, for `compute-sanitizer --tool memcheck` (out-of-bounds / misaligned
accesses show up as errors; sizes are kept small because memcheck slows kernels 10-50x)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rsprompter_b200 import _lib  # noqa: E402

g = torch.Generator().manual_seed(0)
dev = "cuda"
# result-record payload
m = (torch.rand(3, 5, 100, generator=g) > 0.5).to(dev)
bits = _lib.pack_mask_bits(m)
assert torch.equal(_lib.unpack_mask_bits(bits, 100), m)
logits = (torch.randn(4, 16, 16, generator=g) * 3).to(dev)
_lib.mask_paste(logits, 0.5, raw=False, bits=torch.empty(4, 64, 8, dtype=torch.uint8, device=dev))
_lib.query_postprocess(logits, torch.tensor([1, 3], dtype=torch.int32, device=dev), torch.rand(2, device=dev),
                       bits=torch.empty(2, 64, 8, dtype=torch.uint8, device=dev))
# uint8 preprocessing
img = torch.randint(0, 256, (3, 45, 70), generator=g, dtype=torch.uint8).to(dev)
_lib.preprocess_u8(img, torch.empty(3, 64, 96, device=dev), [1., 2., 3.], [4., 5., 6.], True, 0.0)
u8 = torch.randint(0, 256, (2, 3, 64, 64), generator=g, dtype=torch.uint8).to(dev)
_lib.patchify16_u8(u8, [1., 2., 3.], [4., 5., 6.], True)
_lib.patchify16_u8(u8.contiguous(memory_format=torch.channels_last), [1., 2., 3.], [4., 5., 6.], False)
# three-pass attention (grouped GEMM, head split, transpose, softmax)
S, H, hd = 48, 2, 80
qkv = torch.randn(S * S, 3 * H * hd, generator=g).to(torch.bfloat16).to(dev)
rh = (torch.randn(2 * S - 1, hd, generator=g) * 0.2).to(torch.bfloat16).to(dev)
_lib.vit_attention(qkv, rh, rh, 1, S, H, hd)
# flash attention, hd 80 (double-buffered S) and window kernel (48-key rounds)
for S_, n_seq in ((64, 1), (14, 5)):
    qkv = torch.randn(n_seq * S_ * S_, 3 * H * hd, generator=g).to(torch.bfloat16).to(dev)
    rt = (torch.randn(2 * S_ - 1, hd, generator=g) * 0.2).to(torch.bfloat16).to(dev)
    _lib.vit_attention(qkv, rt, rt, n_seq, S_, H, hd)
# layernorm with the bf16 side copy, GroupNorm
x = torch.randn(300, 1280, generator=g).to(dev)
w = torch.ones(1280, device=dev)
_lib.layernorm(x, w, w, 1e-6, copy_out=torch.empty(300, 1280, device=dev, dtype=torch.bfloat16))
xn = torch.randn(2, 24, 16, 128, generator=g).to(torch.bfloat16).to(dev)
_lib.groupnorm_nhwc(xn, torch.ones(128, device=dev), torch.zeros(128, device=dev), 32)
# mask_embed_src (mma path: HW % 128 == 0)
wts = [torch.randn(*s, generator=g).to(dev) for s in ((4, 1, 2, 2), (4,), (4,), (4,), (16, 4, 2, 2), (16,), (16,), (16,), (256, 16), (256,))]
mpp = torch.randn(3, 64, 64, generator=g).to(dev)
_lib.mask_embed_src(mpp, wts, torch.randn(16 * 16, 256, generator=g).to(dev), torch.randn(16 * 16, 256, generator=g).to(dev), 3, (16, 16))
torch.cuda.synchronize()
print("sanitize_small: all launches completed")
