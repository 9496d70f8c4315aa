"""The e4m3 encoder mode against the fp16 mode on the GPU, same process, alternating.

    python tools/bench_fp8.py [--configs tiny,small,medium,large,xlarge] [--rounds 3] [--steps 20] [--warmup 5] [--out FILE]

Per config at its BASELINE batch size (tiny, which BASELINE runs on the CPU only, at 32): images/s of device-resident
synthetic 640x640 batches through the CUDA graph for both modes, alternated, median of `rounds`; batch-1 p50 latency
(CUDA graph, CUDA events); the per-op times (lwdetr_profile_ops) of the encoder's ln1 / qkv / ln2 / fc1 summed over the
blocks in both modes (the fp16 mode with fuse_layernorm = 0, so that its LayerNorms and GEMMs are separate ops as in the
e4m3 mode, and with its default fused schedule for the total), and the e4m3 GEMMs' achieved TFLOP/s against the data
sheet's 1,979 dense FP8 TFLOP/s, named as a ceiling.  The GPU's name, power limit and SM clocks are read in the same run.
Prints one JSON line per config; --out also writes them.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_images, synth_state_dict  # noqa: E402
from bench_resolution import events_ms, gpu_info  # noqa: E402

BATCH = {"tiny": 32, "small": 32, "medium": 64, "large": 32, "xlarge": 16}
FP8_DENSE_TFLOPS = 1979.0        # H100 SXM data sheet, dense FP8: a ceiling, not a measured rate
MODES = {"fp16": torch.float16, "fp8": torch.float8_e4m3fn}


def throughput(eng, xs, steps):
    return len(xs[0]) * steps / (events_ms(lambda i: eng.forward(xs[i & 1], want_aux=False), steps) * 1e-3)


def encoder_ops(eng):
    """{ln1, qkv, ln2, fc1: (ms, flops)} summed over the ViT blocks of the last planned batch."""
    acc = {k: [0.0, 0.0] for k in ("ln1", "qkv", "ln2", "fc1")}
    for label, fl, _, ms in eng.profile_ops(iters=5):
        if label.startswith("block") and "." in label:
            k = label.split(".", 1)[1]
            if k in acc:
                acc[k][0] += ms
                acc[k][1] += fl
    return acc


def run_config(name, rounds, steps, warmup):
    cfg = CONFIGS[name]
    batch = BATCH[name]
    sd = synth_state_dict(cfg, 1)
    xs = [synth_images(batch, 100 + i).cuda() for i in range(2)]
    engs = {}
    for m, dt in MODES.items():
        e = capi.Engine(cfg, dt)
        e.load_state_dict(sd)
        e.set_option("cuda_graph", 1)
        for i in range(warmup):
            e.forward(xs[i & 1], want_aux=False)
        engs[m] = e
    ips = {m: [] for m in MODES}
    for r in range(rounds):                 # alternate the modes within each round
        for m in MODES:
            ips[m].append(throughput(engs[m], xs, steps))
    res = {"config": name, "batch": batch, "images_per_s": {m: statistics.median(v) for m, v in ips.items()},
           "images_per_s_rounds": ips}
    res["speedup"] = res["images_per_s"]["fp8"] / res["images_per_s"]["fp16"]
    # per-op times at the batch size (eager ops, CUDA events)
    ops = {"fp8": encoder_ops(engs["fp8"]), "fp16_fused": encoder_ops(engs["fp16"])}
    tot = {m: sum(o[3] for o in engs[m].profile_ops(iters=3)) for m in MODES}
    sep = capi.Engine(cfg, torch.float16)
    sep.load_state_dict(sd)
    sep.set_option("fuse_layernorm", 0)
    sep.forward(xs[0], want_aux=False)
    ops["fp16_unfused"] = encoder_ops(sep)
    sep.close()
    res["encoder_ops_ms"] = {m: {k: round(v[0], 4) for k, v in o.items()} for m, o in ops.items()}
    res["ops_total_ms"] = {m: round(v, 3) for m, v in tot.items()}
    tf = {}
    for k in ("qkv", "fc1"):
        ms, fl = ops["fp8"][k]
        tf[k] = fl / (ms * 1e-3) / 1e12 if ms > 0 else 0.0
    res["fp8_gemm_tflops"] = {k: round(v, 1) for k, v in tf.items()}
    res["fp8_gemm_share_of_datasheet_ceiling"] = {k: round(v / FP8_DENSE_TFLOPS, 4) for k, v in tf.items()}
    # batch-1 latency
    x1 = synth_images(1, 7).cuda()
    res["b1_p50_ms"] = {}
    for m, e in engs.items():
        for i in range(warmup):
            e.forward(x1, want_aux=False)
        lat = sorted(events_ms(lambda _: e.forward(x1, want_aux=False), 1) for _ in range(max(30, steps)))
        res["b1_p50_ms"][m] = lat[len(lat) // 2]
    for e in engs.values():
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="tiny,small,medium,large,xlarge")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8: needs a CUDA device")
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu}), flush=True)
    rows = []
    for name in a.configs.split(","):
        r = run_config(name, a.rounds, a.steps, a.warmup)
        rows.append(r)
        print(json.dumps(r), flush=True)
    gpu.update({"after_run_" + k: v for k, v in gpu_info().items() if k != "name"})
    print(json.dumps({"gpu_after": gpu}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
