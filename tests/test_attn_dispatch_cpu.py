"""Which attention kernel lwdetr_attention_ex chooses, and what it refuses, without a device (dry runs make no CUDA call).

Coverage: the attn_kernel / attn_short_kernel instances compiled into the shipped library (cuobjdump) must be exactly the
instances the case table of test_attn_mma_gpu.py reaches under LWDETR_B200_ATTN_POLY = 0, 1 and 2, so a new instance cannot
ship without a test that runs it.  Rejections go through dry runs only: the addresses are integers that nothing dereferences."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lw-detr_b200", "lib", "liblwdetr_b200.so")
GPU_TABLE = os.path.join(ROOT, "tests", "test_attn_mma_gpu.py")
DT_NAMES = {"6__half": "float16", "13__nv_bfloat16": "bfloat16"}


@pytest.fixture(scope="module")
def capi():
    if not os.path.exists(LIB):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    from b200 import capi as c
    return c


def _compiled():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    out = set()
    for m in re.finditer(r"Function : _ZN3lwb11attn_kernelI(6__half|13__nv_bfloat16)Li(\d+)ELi(\d+)ELj(\d+)EEEvNS_8AttnArgsE", sass):
        out.add((DT_NAMES[m.group(1)], "mma", int(m.group(2)), int(m.group(3)), int(m.group(4))))
    for m in re.finditer(r"Function : _ZN3lwb17attn_short_kernelI(6__half|13__nv_bfloat16)Li(\d+)ELj(\d+)EEEvNS_8AttnArgsE", sass):
        out.add((DT_NAMES[m.group(1)], "mma_short", int(m.group(2)), 0, int(m.group(3))))
    return out


def test_every_compiled_mma_instance_is_reached_by_the_gpu_table(capi):
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    compiled = _compiled()
    assert len(compiled) == 34, sorted(compiled)             # 2 dtypes x 17 (attn.cu: run_short / run_long)
    reached = set()
    for policy in (0, 1, 2):
        env = dict(os.environ, LWDETR_B200_ATTN_POLY=str(policy), CUDA_VISIBLE_DEVICES="")
        r = subprocess.run([sys.executable, GPU_TABLE, "dry-run"], env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
        reached |= {tuple(x) for x in json.loads(r.stdout.strip().splitlines()[-1])}
    mma = {x for x in reached if x[1] != "wg"}
    print("mma.sync instances covered: %d of %d compiled" % (len(mma & compiled), len(compiled)))
    assert mma == compiled, ("compiled, never run: %s" % sorted(compiled - mma), "run, not compiled: %s" % sorted(mma - compiled))
    assert {x for x in reached if x[1] == "wg"}                # the packed cases still reach the wgmma kernel


A = 1 << 32     # dry-run addresses: never dereferenced


def _dry(capi, q=(A, 256), k=(A + 256, 256), v=(A + (1 << 24), 128), o=(A + (1 << 26), 128), nseq=2, seqlen=300, heads=4, dh=32,
         dtype=torch.float16):
    return capi.attention_ex(q, k, v, o, nseq, seqlen, heads, dh, dh ** -0.5 if dh > 0 else 1.0, dry_run=True, dtype=dtype)


def test_decoder_layout_reports_its_kernel(capi):
    assert _dry(capi) == {"kernel": "mma", "warps": 4, "poly_mask": 0}
    assert _dry(capi, seqlen=100) == {"kernel": "mma_short", "warps": 0, "poly_mask": 0}
    assert _dry(capi, seqlen=1024, dtype=torch.bfloat16) == {"kernel": "mma", "warps": 8, "poly_mask": 0}
    # packed: k = q + C, v = q + 2C, one leading dimension
    assert _dry(capi, q=(A, 384), k=(A + 256, 384), v=(A + 512, 384), seqlen=1600)["kernel"] == "wg"


@pytest.mark.parametrize("which", ["q", "k", "v", "out"])
@pytest.mark.parametrize("off", [2, 8])
def test_misaligned_matrices_are_refused(capi, which, off):
    args = {"q": (A, 256), "k": (A + 256, 256), "v": (A + (1 << 24), 128), "o": (A + (1 << 26), 128)}
    key = "o" if which == "out" else which
    args[key] = (args[key][0] + off, args[key][1])
    for seqlen in (100, 300):
        with pytest.raises(RuntimeError, match="%s must be 16-byte aligned" % which):
            _dry(capi, seqlen=seqlen, **args)
    # the same offset on a packed matrix (all three views move together) is refused as well
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        _dry(capi, q=(A + off, 384), k=(A + off + 256, 384), v=(A + off + 512, 384), seqlen=1600)


@pytest.mark.parametrize("dh", [48, 8, 128, 0])
def test_head_dims_outside_16_32_64_are_refused(capi, dh):
    with pytest.raises(RuntimeError, match="head dim must be 16, 32 or 64"):
        _dry(capi, dh=dh, heads=2)


@pytest.mark.parametrize("field", ["nseq", "seqlen", "heads"])
@pytest.mark.parametrize("value", [0, -1])
def test_non_positive_sizes_are_refused(capi, field, value):
    with pytest.raises(RuntimeError, match="nseq, seqlen and heads must be positive"):
        _dry(capi, **{field: value})


def test_grid_limits_are_refused(capi):
    with pytest.raises(RuntimeError, match="nseq must be at most 65535 .grid z of attn_kernel"):
        _dry(capi, nseq=65536)
    assert _dry(capi, nseq=65535)["kernel"] == "mma"
    assert _dry(capi, nseq=65536, seqlen=100)["kernel"] == "mma_short"      # persistent CTAs: no grid dimension per sequence
    with pytest.raises(RuntimeError, match="nseq must be at most 65535 .grid z of attn_wg_kernel"):
        _dry(capi, q=(A, 384), k=(A + 256, 384), v=(A + 512, 384), nseq=65536, seqlen=100)


def _decoder_layout(heads, dh):
    """q / k column slices of one [*, 2W + 8] matrix, v and out separate (W = heads * dh): the mma.sync path."""
    W = heads * dh
    return dict(q=(A, 2 * W + 8), k=(A + 2 * W, 2 * W + 8), v=(A + (1 << 40), W), o=(A + (1 << 41), W), heads=heads, dh=dh)


def _packed_layout(heads, dh):
    """q / k / v column blocks of one [*, 3W] matrix: the wgmma path."""
    W = heads * dh
    return dict(q=(A, 3 * W), k=(A + 2 * W, 3 * W), v=(A + 4 * W, 3 * W), o=(A + (1 << 41), W), heads=heads, dh=dh)


def test_head_count_grid_limit_is_refused(capi):
    # heads is grid y of attn_kernel and attn_wg_kernel; attn_short_kernel walks (sequence, head) items instead
    with pytest.raises(RuntimeError, match=r"heads must be at most 65535 \(grid y of attn_kernel\)"):
        _dry(capi, **_decoder_layout(65536, 16))
    assert _dry(capi, **_decoder_layout(65535, 16))["kernel"] == "mma"
    assert _dry(capi, seqlen=100, **_decoder_layout(65536, 16))["kernel"] == "mma_short"
    with pytest.raises(RuntimeError, match=r"heads must be at most 65535 \(grid y of attn_wg_kernel\)"):
        _dry(capi, **_packed_layout(65536, 16))
    assert _dry(capi, **_packed_layout(65535, 16))["kernel"] == "wg"


def test_packed_row_count_limit_is_refused(capi):
    # attn_wg_kernel addresses the first row of a sequence as an int TMA coordinate
    with pytest.raises(RuntimeError, match=r"nseq \* seqlen must be below 2\^31"):
        _dry(capi, nseq=65535, seqlen=32769, **_packed_layout(4, 32))         # 2 147 516 415 rows
    assert _dry(capi, nseq=65535, seqlen=32768, **_packed_layout(4, 32))["kernel"] == "wg"    # 2 147 450 880 rows


def test_leading_dimensions_are_refused(capi):
    with pytest.raises(RuntimeError, match="multiples of 8"):
        _dry(capi, v=(A + (1 << 24), 132))
    with pytest.raises(RuntimeError, match="at least heads"):
        _dry(capi, o=(A + (1 << 26), 120))
