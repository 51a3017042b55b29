"""What ptxas made of the wgmma GEMMs (no GPU needed): build the library for sm_90a and read the per-source ptxas
reports the Makefile keeps under csrc/build/.

* No C7510 anywhere: a function call inside a wgmma kernel makes ptxas serialise every wgmma of that kernel (each
  64 x BN x 16 instruction waits for the previous one to retire), which costs the GEMMs a large share of their rate.
* No register spills in the standard-epilogue instantiations of the v2 GEMM, which carry almost every FLOP of the
  encoder."""
import glob
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "rsprompter_b200", "csrc", "build")
ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")
SPILLS = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
V2_STD = re.compile(r"_ZN3rsp2v225gemm_bf16_wgmma_v2_kernelILi(\d+)ELi0EEE")


@pytest.fixture(scope="module")
def ptxas_logs():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import __graft_entry__
    __graft_entry__.build()
    paths = sorted(glob.glob(os.path.join(BUILD, "*.ptxas.log")))
    assert paths, "the build left no ptxas reports"
    logs = {}
    for p in paths:
        with open(p) as f:
            logs[os.path.basename(p)] = f.read()
    return logs


def _spills(text):
    """{kernel: (spill store bytes, spill load bytes)} from one ptxas -v report."""
    out, cur = {}, None
    for line in text.splitlines():
        m = ENTRY.search(line)
        if m:
            cur = m.group(1)
            continue
        m = SPILLS.search(line)
        if m and cur is not None:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


def test_no_serialised_wgmma(ptxas_logs):
    bad = {name: [l for l in text.splitlines() if "C7510" in l][:2] for name, text in ptxas_logs.items()
           if "C7510" in text}
    assert not bad, bad


def test_v2_standard_epilogue_does_not_spill(ptxas_logs):
    spills = _spills(ptxas_logs["gemm_v2.ptxas.log"])
    std = {V2_STD.search(k).group(1): v for k, v in spills.items() if V2_STD.search(k)}
    assert std, "no standard-epilogue instantiation of gemm_bf16_wgmma_v2_kernel in the report"
    bad = {f"BN={bn}": v for bn, v in std.items() if v != (0, 0)}
    assert not bad, f"spill (store, load) bytes: {bad}"
