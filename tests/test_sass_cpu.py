"""The shipped library really takes the Hopper path: SASS mnemonic counts per kernel (cuobjdump, no GPU needed).
HGMMA = wgmma.mma_async, UTMALDG = TMA tensor load, UBLKCP = cp.async.bulk, HMMA = mma.sync, LDGSTS = cp.async."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lw-detr_b200", "lib", "liblwdetr_b200.so")


@pytest.fixture(scope="module")
def table():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    if not os.path.exists(LIB):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_proof.py"), LIB], capture_output=True, text=True, check=True).stdout
    rows, cols = {}, None
    for line in out.splitlines():
        if line.startswith("#"):
            continue
        if line.startswith("kernel"):
            cols = line.split()[1:]
            continue
        m = re.match(r"(.*?)\s+((?:\d+\s*)+)$", line)
        if m and cols:
            vals = [int(v) for v in m.group(2).split()]
            if len(vals) == len(cols):
                rows[m.group(1).strip()] = dict(zip(cols, vals))
    assert rows, out[:500]
    return rows


def _sel(table, prefix):
    return {k: v for k, v in table.items() if prefix in k}


def test_packed_attention_kernels_are_wgmma_tma_only(table):
    ks = _sel(table, "attn_wg_kernel<")
    assert len(ks) >= 6                      # head dims 16 / 32 / 64 in fp16 and bf16
    for name, c in ks.items():
        assert c["HGMMA"] > 0 and c["UTMALDG"] > 0 and c["SYNCS"] > 0, name
        assert c["HMMA"] == 0 and c["LDGSTS"] == 0, name


def test_gemm_family_is_wgmma_tma(table):
    ks = _sel(table, "gemm_tc_kernel<")
    assert len(ks) >= 24
    for name, c in ks.items():
        assert c["HGMMA"] > 0 and c["UTMALDG"] > 0 and c["SYNCS"] > 0, name
        assert c["HMMA"] == 0 and c["LDGSTS"] == 0, name


def test_deformable_gather_streams_with_bulk_copies(table):
    ks = _sel(table, "msda_fwd_kernel<")
    assert ks
    for name, c in ks.items():
        assert c["UBLKCP"] > 0 and c["SYNCS"] > 0, name


def test_legacy_mma_sync_only_where_documented(table):
    """mma.sync (HMMA) is allowed only in attn.cu's kernels: decoder self-attention, unpacked q/k/v."""
    for name, c in table.items():
        if c["HMMA"] > 0:
            assert name.startswith("attn_kernel<") or name.startswith("attn_short_kernel<"), name
