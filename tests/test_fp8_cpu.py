"""The e4m3 encoder mode without a GPU: the host weight quantiser bit for bit, the mode's CPU spec (tools/oracle_fp8.py)
and what its quantisation costs against the fp32 oracle, the C ABI's handling of the mode, and the FP8 GEMM's SASS."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import oracle_fp8  # noqa: E402

# Quantisation cost of the e4m3 scheme against the fp32 oracle on the synthetic weights (weight seed 1, image seed 0, B = 2,
# 640 x 640), measured on the CPU (deterministic): T1 worst tap rel-L2, T2 logits rel-L2 and boxes max-abs with the
# two-stage indices forced to the fp32 oracle's, T3 smallest per-image set agreement.  DESIGN.md section 4 lists them.
COST = {
    "tiny": dict(tap_rel_l2=0.01185, logits_rel_l2=0.004556, boxes_maxabs=0.002455, set_agreement_min=0.98),
    "small": dict(tap_rel_l2=0.01537, logits_rel_l2=0.005002, boxes_maxabs=0.002699, set_agreement_min=0.9867),
    "medium": dict(tap_rel_l2=0.01524, logits_rel_l2=0.005091, boxes_maxabs=0.001672, set_agreement_min=0.9767),
    "large": dict(tap_rel_l2=0.01523, logits_rel_l2=0.005378, boxes_maxabs=0.003573, set_agreement_min=0.98),
    "xlarge": dict(tap_rel_l2=0.01514, logits_rel_l2=0.004780, boxes_maxabs=0.003566, set_agreement_min=0.9833),
}


def _lib():
    from b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return capi


def _rows_cases():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(40, 256, generator=g) * 3
    x[1] = 0.0                                                   # all-zero row: scale 1, codes 0
    x[2] = torch.randint(-4, 5, (256,), generator=g).float()     # max exactly 4: 448 / 4 exact
    x[3] = -x[3].abs()                                           # all negative
    x[4] = 0.0
    x[4, 0] = 448.0
    x[4, 1:] = torch.rand(255, generator=g) * 0.03               # most of the row in e4m3's subnormal range after scaling
    x[5] = torch.linspace(-1, 1, 256) * 1e-30                    # tiny magnitudes
    x[6, :] = 1.0
    x[6, 7] = -1.0                                               # ties of |x|
    return x


def test_host_quantiser_is_bit_identical_to_the_torch_restatement():
    capi = _lib()
    x = _rows_cases()
    q, s = capi.host_quant_e4m3_rows(x)
    qt, st = oracle_fp8.quant_rows(x)
    assert torch.equal(q, qt.view(torch.uint8))
    assert torch.equal(s, st[:, 0])
    assert torch.equal(q[1], torch.zeros(256, dtype=torch.uint8)) and s[1].item() == 1.0
    assert (q[4, 1:] & 0x78 == 0).any()                          # some subnormal codes were produced
    assert ((q[3] & 0x80) != 0)[x[3] != 0].all()                 # negative values keep their sign bit
    assert q[4, 0].item() == 0x7E                                # the row maximum is 448


def test_unquantised_composition_is_the_oracle():
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    from oracle import lwdetr_oracle as orc
    cfg = CONFIGS["tiny"]
    sd = synth_state_dict(cfg, 1)
    x = synth_images(2, 0)
    a = orc.forward(sd, cfg, x)
    b = oracle_fp8.forward(sd, cfg, x, quantize=False)
    for k in ("pred_logits", "pred_boxes"):
        assert (a[k] - b[k]).abs().max().item() <= 1e-6, k
    assert (a["enc_outputs"]["pred_boxes"] - b["enc_outputs"]["pred_boxes"]).abs().max().item() <= 1e-6


@pytest.mark.parametrize("name", list(COST))
def test_quantisation_cost_against_the_fp32_oracle(name):
    """A change of the e4m3 scheme (or of the synthetic weights) shows up here: each statistic within 5 % of the value
    recorded in DESIGN.md section 4 (set agreement within one query of it)."""
    got = oracle_fp8.quant_cost(name, batch=2)
    want = COST[name]
    print(name, got)
    for k in ("tap_rel_l2", "logits_rel_l2", "boxes_maxabs"):
        assert abs(got[k] - want[k]) <= 0.05 * want[k], (k, got[k], want[k])
    assert abs(got["set_agreement_min"] - want["set_agreement_min"]) <= 0.011, got


def test_create_in_the_e4m3_mode_fails_cleanly_without_a_gpu():
    capi = _lib()
    from b200.config import CONFIGS
    cs = capi.config_struct(CONFIGS["tiny"])
    h = ctypes.c_void_p()
    if not torch.cuda.is_available():
        assert capi.lib().lwdetr_create(ctypes.byref(cs), capi.F16_E4M3, ctypes.byref(h)) != 0
        assert "no CUDA device" in capi.lib().lwdetr_last_error().decode()
    assert capi.lib().lwdetr_create(ctypes.byref(cs), 3, ctypes.byref(h)) != 0
    assert "LWDETR_F16_E4M3" in capi.lib().lwdetr_last_error().decode()
    assert capi.dtype_code(torch.float8_e4m3fn) == capi.F16_E4M3
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        capi.kernel_dtype_code(torch.float8_e4m3fn)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        capi.dtype_code(torch.float32)


def test_kernel_level_gemm_rejects_the_e4m3_code():
    """lwdetr_gemm (16-bit) refuses dtype 2 before touching any pointer: e4m3 GEMMs go through lwdetr_gemm_e4m3."""
    capi = _lib()
    dummy = ctypes.c_void_p(16)
    rc = capi.lib().lwdetr_gemm(capi.F16_E4M3, dummy, 64, 1, 64, dummy, 64, None, None, None, 0, 0, 0, dummy, 64, 0, 0, 0, 0, 0, 0, None)
    assert rc != 0 and "fp16 or bf16" in capi.lib().lwdetr_last_error().decode()
    rc = capi.lib().lwdetr_gemm_e4m3(dummy, 64, dummy, 1, 96, dummy, dummy, 64, None, 0, dummy, 64, None)
    assert rc != 0 and "multiple of 64" in capi.lib().lwdetr_last_error().decode()


def test_fp8_gemm_is_qgmma_tma():
    import shutil
    import subprocess
    import re
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    capi = _lib()
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
    ks = {k: v for k, v in rows.items() if k.startswith("gemm_e4m3_kernel<")}
    assert len(ks) == 8                                          # BN 64 / 128 / 192 / 256, GELU on / off
    for name, c in ks.items():
        assert c["QGMMA"] > 0 and c["UTMALDG"] > 0 and c["SYNCS"] > 0, name
        assert c["HMMA"] == 0 and c["HGMMA"] == 0, name
    for name, c in rows.items():
        if name.startswith("gemm_tc_kernel<"):
            assert c["QGMMA"] == 0, name
