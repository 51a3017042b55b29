"""What ptxas made of the wgmma ViT attention kernel (no GPU needed): build the library for sm_90a and read the
attention report the Makefile keeps under csrc/build/.  Every instantiation must be free of register spills: the
consumer warpgroups hold the score, output and P fragments in registers, and a spill there lands inside the
softmax between two wgmmas."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "attention.ptxas.log")
ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
KERNEL = re.compile(r"_ZN3rsp20vit_attention_kernelILi(\d+)ELi(\d+)EEE")


@pytest.fixture(scope="module")
def attention_log():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(LOG) as f:
        return f.read()


def test_attention_kernel_does_not_spill(attention_log):
    spills, cur = {}, None
    for line in attention_log.splitlines():
        m = ENTRY.search(line)
        if m:
            cur = m.group(1)
            continue
        m = SPILLS.search(line)
        if m and cur is not None:
            k = KERNEL.search(cur)
            if k:
                spills[(int(k.group(1)), int(k.group(2)))] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert set(spills) == {(hd, s) for hd in (64, 80) for s in (14, 32, 64)}, sorted(spills)
    bad = {f"hd={hd} S={s}": v for (hd, s), v in spills.items() if v != (0, 0)}
    assert not bad, f"spill (store, load) bytes: {bad}"
