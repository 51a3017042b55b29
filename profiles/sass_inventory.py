"""Per-kernel SASS inventory of librsp_b200.so: counts of the Hopper mnemonics that prove which hardware path a
kernel uses (HGMMA = wgmma, HMMA = mma.sync, UTMALDG/UTMASTG = TMA load/store, LDSM = ldmatrix, LDGSTS = cp.async,
SYNCS = mbarrier, MUFU.EX2 = exp2).  Usage: python profiles/sass_inventory.py [out.txt]"""
import collections
import re
import subprocess
import sys

LIB = "rsprompter_b200/librsp_b200.so"
PATS = ["HGMMA", "HMMA", "UTMALDG", "UTMASTG", "LDSM", "LDGSTS", "SYNCS", "MUFU.EX2"]


def main(out=None):
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        for p in PATS:
            if re.search(r"\b" + re.escape(p), line):
                counts[cur][p] += 1
        if re.match(r"\s*/\*[0-9a-f]{4}\*/", line):
            counts[cur]["instr"] += 1
    dem = subprocess.run(["cu++filt"], input="\n".join(counts), capture_output=True, text=True).stdout.splitlines()
    rows = []
    for (k, c), name in zip(counts.items(), dem):
        name = re.sub(r"\((int|bool)\)", "", name.replace("void ", "").replace("rsp::", ""))
        name = re.sub(r"\(.*", "", name)
        rows.append((name, c))
    lines = ["%-78s %7s " % ("kernel", "instr") + " ".join("%8s" % p for p in PATS)]
    for name, c in sorted(rows, key=lambda r: -r[1]["UTCHMMA"] * 10 ** 6 - r[1]["instr"]):
        lines.append("%-78s %7d " % (name[:78], c["instr"]) + " ".join("%8d" % c[p] for p in PATS))
    text = "\n".join(lines)
    print(text)
    if out:
        with open(out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main(*sys.argv[1:2])
