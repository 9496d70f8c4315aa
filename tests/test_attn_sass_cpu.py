"""The packed-qkv attention kernel at head dims 16 and 32 as compiled for sm_90a (cuobjdump, no GPU needed): its MMAs are
wgmma, a short tail chunk takes the 40-key form, and it neither spills nor exceeds the register budget of the resident
CTAs it is built for (attn_wg.cu: kMinCtas)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lw-detr_b200", "lib", "liblwdetr_b200.so")
REGS_PER_SM, THREADS = 65536, 288
MIN_CTAS = {16: 3, 32: 2}


@pytest.fixture(scope="module")
def kernels():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    if not os.path.exists(LIB):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    out = {}
    for dt in ("6__half", "13__nv_bfloat16"):
        for dh in (16, 32):
            tag = "attn_wg_kernelI%sLi%dE" % (dt, dh)
            m = re.search(r"Function : (\S*%s\S*)\n(.*?)(?=\n\s*Function : |\Z)" % re.escape(tag), sass, re.S)
            assert m, tag
            ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Za-z0-9_.]+)", m.group(2))
            r = re.search(r"Function %s:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)" % re.escape(m.group(1)), res)
            assert r, tag
            out[(dt, dh)] = {"ops": ops, "reg": int(r.group(1)), "stack": int(r.group(2)), "local": int(r.group(3))}
    return out


def test_mmas_are_wgmma_with_a_40_key_tail(kernels):
    for key, k in kernels.items():
        assert any(op.startswith("HGMMA.64x64x16") for op in k["ops"]), key    # S of a 64-key chunk
        assert any(op.startswith("HGMMA.64x40x16") for op in k["ops"]), key    # S of a tail of <= 40 keys
        assert not any(op.startswith("HMMA") for op in k["ops"]), key


def test_nothing_spills(kernels):
    for key, k in kernels.items():
        assert not any(op.startswith(("STL", "LDL")) for op in k["ops"]), key
        assert k["stack"] == 0 and k["local"] == 0, key


def test_register_budget_allows_the_resident_ctas(kernels):
    for (dt, dh), k in kernels.items():
        regs = (k["reg"] + 7) // 8 * 8                              # allocated per thread in units of 8
        assert regs * THREADS * MIN_CTAS[dh] <= REGS_PER_SM, (dt, dh, k["reg"])
