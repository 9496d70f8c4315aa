"""Throughput and latency of the CUDA path at several input sizes (lwdetr_forward_hw).

    python tools/bench_resolution.py [--configs tiny,small,...] [--sizes 640x640,448x768,1024x1024,768x1344]
                                     [--batch 8] [--dtype fp16] [--steps 20] [--warmup 5] [--out FILE]

Per (config, size): images/s of device-resident synthetic batches through the CUDA graph, batch-1 p50 latency (CUDA
graph, CUDA events), and the most expensive ops of the schedule (CUDA events per op, lwdetr_profile_ops) with the
deformable-attention and top-k ops always listed.  The GPU's name, power limit and SM clocks are read in the same run.
Prints one JSON line per (config, size); --out also writes the list as JSON.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_images, synth_state_dict  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = "power.limit,clocks.sm,clocks.max.sm"
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        info.update(dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")])))
    except (OSError, subprocess.SubprocessError):
        info["nvidia_smi"] = "not available"
    return info


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def measure(eng, name, H, W, batch, steps, warmup, top):
    xs = [synth_images(batch, 100 + i, (H, W)).cuda() for i in range(2)]
    step = lambda i: eng.forward(xs[i & 1], want_aux=False)
    for i in range(warmup):
        step(i)
    ms = events_ms(step, steps)
    res = {"config": name, "hw": [H, W], "batch": batch, "tokens": (H // 16) * (W // 16),
           "memory_len": CONFIGS[name].memory_len_at(H, W), "images_per_s": batch * steps / (ms * 1e-3)}
    # per-op times of the batch schedule (the eager ops, CUDA events around `iters` launches of each)
    ops = eng.profile_ops(iters=5)
    total = sum(o[3] for o in ops)
    ranked = sorted(ops, key=lambda o: -o[3])
    keep = [o for o in ranked[:top]] + [o for o in ops if (o[0].endswith(".msda") or o[0] == "topk") and o not in ranked[:top]]
    res["ops_total_ms"] = total
    res["top_ops"] = [{"op": o[0], "ms": round(o[3], 4), "share": round(o[3] / total, 4)} for o in keep]
    # batch-1 latency: a new plan (B = 1), graph captured after the eager first run
    x1 = synth_images(1, 7, (H, W)).cuda()
    for i in range(warmup):
        eng.forward(x1, want_aux=False)
    lat = []
    for i in range(max(20, steps)):
        lat.append(events_ms(lambda _: eng.forward(x1, want_aux=False), 1))
    lat.sort()
    res["b1_p50_ms"] = lat[len(lat) // 2]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="tiny,small,medium,large,xlarge")
    ap.add_argument("--sizes", default="640x640,448x768,1024x1024,768x1344")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--top", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resolution: needs a CUDA device")
    dt = {"fp16": torch.float16, "bf16": torch.bfloat16}[a.dtype]
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu, "dtype": a.dtype}), flush=True)
    rows = []
    for name in a.configs.split(","):
        cfg = CONFIGS[name]
        eng = capi.Engine(cfg, dt)
        eng.load_state_dict(synth_state_dict(cfg, 1))
        eng.set_option("cuda_graph", 1)
        for s in a.sizes.split(","):
            H, W = (int(v) for v in s.lower().split("x"))
            r = measure(eng, name, H, W, a.batch, a.steps, a.warmup, a.top)
            r["dtype"] = a.dtype
            rows.append(r)
            print(json.dumps(r), flush=True)
        eng.close()
    gpu.update({"after_run_" + k: v for k, v in gpu_info().items() if k != "name"})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
