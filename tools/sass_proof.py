"""Per-kernel counts of the SASS mnemonics that prove which hardware path a kernel takes, from `cuobjdump -sass` of the
shipped library (runs without a GPU).
    python tools/sass_proof.py [lib]
A function's block runs from its "Function : <mangled>" line to the next one; every instruction line of the block is counted
(a block does not end at its first blank line: long kernels contain several)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = ["HGMMA", "UTMALDG", "UBLKCP", "HMMA", "MUFU.EX2", "LDGSTS", "LDSM", "SYNCS", "QGMMA"]


def main(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", out)), capture_output=True, text=True).stdout.split("\n")
    counts, order, cur, k = {}, [], None, 0
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = names[k].strip() if k < len(names) else m.group(1)
            k += 1
            cur = re.sub(r"\(.*$", "", cur).replace("void lwb::", "").replace("lwb::", "").replace("(anonymous namespace)::", "")
            cur = re.sub(r"\((int|bool|unsigned int)\)", "", cur)
            counts[cur] = collections.Counter()
            order.append(cur)
            continue
        if cur is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not m:
            continue
        op = m.group(1)
        for c in COLS:
            if op == c or op.startswith(c + "."):
                counts[cur][c] += 1
    print("# cuobjdump -sass %s (sm_90a): per-kernel counts of the SASS mnemonics that prove the path" % os.path.relpath(lib, ROOT))
    print("# HGMMA = wgmma.mma_async, UTMALDG = TMA tensor load, UBLKCP = cp.async.bulk (1-D bulk copy), HMMA = mma.sync,")
    print("# LDGSTS = cp.async, LDSM = ldmatrix, SYNCS = mbarrier operations, QGMMA = FP8 wgmma.mma_async")
    w = max(len(n) for n in order) + 2
    print("%-*s" % (w, "kernel") + "".join("%11s" % c for c in COLS))
    for n in sorted(order):
        print("%-*s" % (w, n) + "".join("%11d" % counts[n][c] for c in COLS))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "lw-detr_b200", "lib", "liblwdetr_b200.so"))
