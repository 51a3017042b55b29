"""What ptxas made of the 128 x 256 standard-epilogue GEMM (EPI_STD_WIDE, no GPU needed): its 128 accumulator
registers per thread stay in registers through the epilogue, so any spill or serialised wgmma shows in the report.

* no C7510 (serialised wgmma) and no spill stores or loads;
* the launch register count fits the setmaxnreg budget of the 384-thread block: ptxas must allocate at most 168 per
  thread, so that 40 for the producer warpgroup and 232 for each MMA warpgroup (3 x 168 in all) are available."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "rsprompter_b200", "csrc", "build", "gemm_v2.ptxas.log")
WIDE = "_ZN3rsp2v225gemm_bf16_wgmma_v2_kernelILi256ELi7EEE"


@pytest.fixture(scope="module")
def wide_report():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    with open(LOG) as f:
        lines = f.read().splitlines()
    start = [i for i, l in enumerate(lines) if "Compiling entry function" in l and WIDE in l]
    assert start, "no EPI_STD_WIDE instantiation of gemm_bf16_wgmma_v2_kernel in the report"
    i = start[0] + 1
    block = []
    while i < len(lines) and "Compiling entry function" not in lines[i]:
        block.append(lines[i])
        i += 1
    return "\n".join(block)


def test_wide_no_serialised_wgmma(wide_report):
    assert "C7510" not in wide_report


def test_wide_does_not_spill(wide_report):
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", wide_report)
    assert m, wide_report
    assert (int(m.group(1)), int(m.group(2))) == (0, 0)


def test_wide_registers_fit_setmaxnreg_budget(wide_report):
    m = re.search(r"Used (\d+) registers", wide_report)
    assert m, wide_report
    regs = int(m.group(1))
    assert regs <= 168 and 40 + 2 * 232 <= 3 * regs, regs
