"""Isolated kernel timings for the two kernels BASELINE.json singles out (deformable-attention gather and
window attention) plus global attention, at the BASELINE configs, through the C ABI.

Timing: CUDA events around each launch, L2 flushed (256 MB write) before every timed launch, median of
`--iters`; achieved = SURVEY.md 8d algorithmic bytes / time, peak = the H100 SXM data sheet's HBM bandwidth (a ceiling).
    python tools/bench_kernels.py --out kernels.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402


def peaks():
    """H100 SXM data sheet (700 W card): HBM3 GB/s, dense 16-bit TFLOP/s - ceilings, not rates this project reached."""
    return 3350.0, 989.0, "H100 SXM data sheet"


def sm_clock_ghz():
    """SM clock of the current device now (nvidia-smi), in GHz; NaN when it cannot be read.  Read right after a timed
    kernel, it sets that kernel's MUFU ceiling: 16 ex2 per clock per SM."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, check=True).stdout
        return float(out.strip().splitlines()[0]) / 1e3
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return float("nan")


FLUSH_MODE = "clean"


def timed(fn, iters, flush):
    """L2 flush before every timed launch.  "dirty": a 256 MB read-modify-write leaves the 50 MB L2 full of DIRTY lines, so
    every line the timed kernel then allocates first evicts a dirty one - the kernel's DRAM reads compete 1:1 with
    write-backs of the flush buffer, which caps a read-only kernel near half of the copy bandwidth.  "clean" (default): the write pass is followed by a
    256 MB read pass of a second buffer, so the L2 holds clean lines of unrelated data: inputs still come from DRAM, and
    only the kernel's own traffic is on the memory bus.  Both are recorded (`flush` field)."""
    ts = []
    for _ in range(3):
        fn()
    for _ in range(iters):
        flush[0].add_(1)                                 # 256 MB read+write evicts the 50 MB L2
        if FLUSH_MODE == "clean":
            flush[1].sum()                               # 256 MB read: what stays in L2 is clean
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    return statistics.median(ts), min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    ap.add_argument("--flush", default="clean", choices=["clean", "dirty"], help="state of the L2 before each timed launch (see timed())")
    ap.add_argument("--only", default=None, help="comma list of kernels: msda_forward,window_attention,global_attention")
    ap.add_argument("--configs", default=None, help="comma list of configs (default: the four BASELINE configs)")
    a = ap.parse_args()
    hbm, tflops, src = peaks()
    global FLUSH_MODE
    FLUSH_MODE = a.flush
    flush = [torch.zeros(64 * 1024 * 1024, device="cuda", dtype=torch.float32) for _ in range(2)]
    res = []
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(0)
    cases = [("small", 32, torch.float16), ("medium", 64, torch.bfloat16), ("large", 32, torch.float16), ("xlarge", 16, torch.float16)]
    only = set(a.only.split(",")) if a.only else None
    if a.configs:
        cases = [c for c in cases if c[0] in a.configs.split(",")]
    for name, B, dt in cases:
        cfg = CONFIGS[name]
        d, M, L, P, nq, S = cfg.hidden_dim, cfg.ca_nheads, cfg.n_levels, cfg.dec_n_points, cfg.num_queries, cfg.memory_len
        # ---- deformable attention core (one decoder layer)
        value = torch.randn(B, 3, M, S, 16, device="cuda", generator=g).to(dt)      # head-major, three layers' values in one buffer
        ol = (torch.randn(B * nq, 3 * M * L * P, device="cuda", generator=g) * 1.5).to(dt)
        ref = torch.rand(B * nq, 4, device="cuda", generator=g) * torch.tensor([0.9, 0.9, 0.4, 0.4], device="cuda") + 0.05
        out = torch.empty(B * nq, d, device="cuda", dtype=dt)
        fn = lambda: capi.msda_forward(value[:, 1], ol, ref, out, B, S, nq, M, L, P, list(cfg.level_shapes), v_image_stride=3 * M * S * 16)
        med, best = timed(fn, a.iters, flush) if (only is None or "msda_forward" in only) else (float("nan"), float("nan"))
        elt = 2
        algo = min(B * S * d, B * nq * M * L * P * 4 * 16) * elt + B * nq * M * L * P * 3 * elt + B * nq * d * elt
        res.append({"kernel": "msda_forward", "config": "%s B=%d %s" % (name, B, str(dt)[6:]), "us_median": med, "us_best": best,
                    "algorithmic_MB": algo / 1e6, "achieved_GBps": algo / med / 1e3, "peak_GBps": hbm, "frac": algo / med / 1e3 / hbm, "bound": "hbm"})
        # ---- ViT attention cores
        C, heads = cfg.vit_dim, cfg.vit_heads
        dh = C // heads
        T = cfg.tokens
        qkv = torch.randn(B * T, 3 * C, device="cuda", generator=g).to(dt)
        att = torch.empty(B * T, C, device="cuda", dtype=dt)
        for kind, nseq, seqlen in (("window_attention", 16 * B, T // 16), ("global_attention", B, T)):
            if only is not None and kind not in only:
                continue
            fn = lambda: capi.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], att, nseq, seqlen, heads, dh, dh ** -0.5)
            med, best = timed(fn, a.iters, flush)
            clk = sm_clock_ghz()
            algo = B * T * 4 * C * elt
            flops = 4.0 * nseq * seqlen * seqlen * C
            exps = nseq * heads * seqlen * seqlen
            r = {"kernel": kind, "config": "%s B=%d %s dh=%d" % (name, B, str(dt)[6:], dh), "us_median": med, "us_best": best,
                 "algorithmic_MB": algo / 1e6, "achieved_GBps": algo / med / 1e3, "peak_GBps": hbm, "hbm_frac": algo / med / 1e3 / hbm,
                 "gflop": flops / 1e9, "achieved_TFLOPs": flops / med / 1e6, "tensor_frac": flops / med / 1e6 / tflops,
                 "gexp_per_s": exps / med / 1e3, "sm_clock_ghz": clk, "exp_frac_of_mufu_peak": exps / med / 1e3 / (16 * sms * clk)}
            r["bound"] = "hbm" if kind == "window_attention" else "tensor (nominal) / exp"
            r["frac"] = r["hbm_frac"] if kind == "window_attention" else r["tensor_frac"]
            res.append(r)
        del value, ol, qkv, att
    for r in res:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"peak_source": src, "timing": "CUDA events, L2 flushed (%s) before each launch, median of %d" % (a.flush, a.iters), "flush": a.flush, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
