"""What ptxas made of the mask decoder's fused wgmma kernels (no GPU needed): build the library for sm_90a and read the
decoder report the Makefile keeps under csrc/build/.  The fused t2i kernel keeps a 64 x 128 wgmma accumulator live
while the same warps run the attention step of the previous tile, and the fused i2t kernel holds a 64 x 256 one
through its LayerNorm, so a spill or a serialised wgmma (C7510 / C7512) there would put local-memory traffic or a
full wgmma drain inside every tile."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "decoder.ptxas.log")
ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
FUSED = ("t2i_fused_kernel", "i2t_fused_kernel")


@pytest.fixture(scope="module")
def decoder_log():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(LOG) as f:
        return f.read()


def test_fused_decoder_kernels_do_not_spill(decoder_log):
    spills, cur = {}, None
    for line in decoder_log.splitlines():
        m = ENTRY.search(line)
        if m:
            cur = m.group(1)
            continue
        m = SPILLS.search(line)
        if m and cur is not None:
            for k in FUSED:
                if k in cur:
                    spills[k] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert set(spills) == set(FUSED), sorted(spills)
    bad = {k: v for k, v in spills.items() if v != (0, 0)}
    assert not bad, f"spill (store, load) bytes: {bad}"


def test_fused_decoder_kernels_keep_wgmma_pipelined(decoder_log):
    bad = [ln for ln in decoder_log.splitlines() if "C751" in ln or "serializ" in ln.lower()]
    assert not bad, bad
