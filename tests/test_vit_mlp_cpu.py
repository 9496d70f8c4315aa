"""The fused ViT MLP without a GPU: its kernels are wgmma + TMA + mbarrier code (SASS), with no mma.sync."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_vit_mlp_kernel_is_hgmma_tma():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))
    from b200 import capi
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_proof.py"), capi.LIB_PATH], capture_output=True,
                         text=True, check=True).stdout
    cols, rows = None, {}
    for line in out.splitlines():
        if line.startswith("kernel"):
            cols = line.split()[1:]
        elif cols and not line.startswith("#"):
            m = re.match(r"(.*?)\s+((?:\d+\s*)+)$", line)
            if m:
                rows[m.group(1).strip()] = dict(zip(cols, [int(v) for v in m.group(2).split()]))
    ks = {k: v for k, v in rows.items() if "vit_mlp_kernel<" in k}
    assert len(ks) == 2, sorted(rows)                            # fp16, bf16
    for name, c in ks.items():
        assert c["HGMMA"] > 0 and c["UTMALDG"] > 0 and c["SYNCS"] > 0, name
        assert c["HMMA"] == 0, name
