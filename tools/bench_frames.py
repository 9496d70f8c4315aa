"""End-to-end rate of detection from raw camera frames: resize on the device (forward_frames) against resize on the host.

    python tools/bench_frames.py [--cases small:32,xlarge:16] [--sources 480x640,720x1280,1080x1920] [--dtype fp16]
                                 [--steps 20] [--warmup 5] [--rounds 3] [--out FILE]

Per (config, batch, source size), pinned host uint8 frames going to 640x640, the four paths alternating in one process:
  frames        forward_frames: H2D copy of the RAW RGB frames + resize fused into the patch gather + forward
  frames_nv12   the same from packed NV12 frames [B, 3h/2, w] (1.5 bytes per pixel), colorspace="bt709": the colour
                conversion is fused into the resize's staging
  u8_ceiling    the existing uint8 path fed frames that are already 640x640 (H2D of those + forward): no resize anywhere
  host_resize   torch's CPU antialias interpolate (all cores) to 640x640, then u8_ceiling's path: what callers do today
Each is images/s by a host clock around `steps` batches ending in a device synchronise; the median of `rounds` is reported
with the spread.  Also the resize op's own time (CUDA events around repeated launches of the patch_gather op of the
schedule, lwdetr_profile_ops) with the bytes it has to move (sum h*w*3 read + B*T*768*2 written) and the time those bytes
take at the H100 SXM data sheet's 3.35 TB/s, named as a floor, not as something reached; and the H2D copy time of the raw
frames.  The same resize-op and copy figures for the NV12 frames (h*w*1.5 bytes read).  The GPU's name and power limit are
read in the same run.  One JSON line per case; --out also writes the list.
Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402
from bench_resolution import events_ms, gpu_info  # noqa: E402

HBM_DATASHEET_BYTES_PER_S = 3.35e12      # H100 SXM data sheet, a card allowed up to 700 W
RUN = 640


def host_rate(step, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(i)
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def measure(eng, name, batch, h, w, steps, warmup, rounds):
    g = torch.Generator().manual_seed(h * 10000 + w)
    raw = [torch.randint(0, 256, (batch, h, w, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    small = [torch.randint(0, 256, (batch, RUN, RUN, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    staged = torch.empty(batch, RUN, RUN, 3, dtype=torch.uint8).pin_memory()
    nv12 = [torch.randint(0, 256, (batch, h * 3 // 2, w), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]

    def frames(i):
        eng.forward_frames(raw[i & 1].cuda(non_blocking=True), want_aux=False)

    def frames_nv12(i):
        eng.forward_frames(nv12[i & 1].cuda(non_blocking=True), want_aux=False, colorspace="bt709")

    def ceiling(i):
        eng.forward(small[i & 1].cuda(non_blocking=True), want_aux=False)

    def host_resize(i):
        x = raw[i & 1].permute(0, 3, 1, 2).float()
        y = F.interpolate(x, size=(RUN, RUN), mode="bilinear", align_corners=False, antialias=True)
        staged.copy_(y.add_(0.5).clamp_(0, 255).to(torch.uint8).permute(0, 2, 3, 1))
        eng.forward(staged.cuda(non_blocking=True), want_aux=False)
        torch.cuda.synchronize()                      # `staged` is reused by the next step

    paths = {"frames": frames, "frames_nv12": frames_nv12, "u8_ceiling": ceiling, "host_resize": host_resize}
    for fn in paths.values():
        for i in range(warmup):
            fn(i)
    rates = {k: [] for k in paths}
    for _ in range(rounds):                           # alternate the paths: other work shares the host and the card
        for k, fn in paths.items():
            rates[k].append(batch * host_rate(fn, steps if k != "host_resize" else max(3, steps // 4)))
    res = {"config": name, "batch": batch, "source": [h, w], "run_size": [RUN, RUN]}
    for k, v in rates.items():
        v.sort()
        res[k + "_images_per_s"] = round(v[len(v) // 2], 1)
        res[k + "_images_per_s_min_max"] = [round(v[0], 1), round(v[-1], 1)]
    # the resize op alone: CUDA events around repeated launches of the schedule's patch_gather op on the last frames batch
    dev = raw[0].cuda()
    eng.forward_frames(dev, want_aux=False)
    op_ms = [o[3] for o in eng.profile_ops(iters=20) if o[0] == "patch_gather"][0]
    moved = batch * h * w * 3 + batch * (RUN // 16) ** 2 * 768 * 2
    res["resize_op_ms"] = round(op_ms, 4)
    res["resize_op_bytes"] = moved
    res["resize_op_GBps"] = round(moved / (op_ms * 1e-3) / 1e9, 1)
    res["resize_op_floor_ms_at_datasheet_3.35TBps"] = round(moved / HBM_DATASHEET_BYTES_PER_S * 1e3, 4)
    res["h2d_raw_frames_ms"] = round(events_ms(lambda i: raw[i & 1].cuda(non_blocking=True), 10) / 10, 4)
    eng.forward_frames(nv12[0].cuda(), want_aux=False, colorspace="bt709")
    op_ms = [o[3] for o in eng.profile_ops(iters=20) if o[0] == "patch_gather"][0]
    moved = batch * h * w * 3 // 2 + batch * (RUN // 16) ** 2 * 768 * 2
    res["nv12_resize_op_ms"] = round(op_ms, 4)
    res["nv12_resize_op_bytes"] = moved
    res["nv12_resize_op_GBps"] = round(moved / (op_ms * 1e-3) / 1e9, 1)
    res["nv12_resize_op_floor_ms_at_datasheet_3.35TBps"] = round(moved / HBM_DATASHEET_BYTES_PER_S * 1e3, 4)
    res["h2d_nv12_frames_ms"] = round(events_ms(lambda i: nv12[i & 1].cuda(non_blocking=True), 10) / 10, 4)
    eng.forward(small[0].cuda(), want_aux=False)
    res["u8_gather_op_ms"] = round([o[3] for o in eng.profile_ops(iters=20) if o[0] == "patch_gather"][0], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="small:32,xlarge:16")
    ap.add_argument("--sources", default="480x640,720x1280,1080x1920")
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames.py needs a CUDA device (an H100); nothing is measured without one")
    dt = {"fp16": torch.float16, "bf16": torch.bfloat16}[a.dtype]
    torch.set_num_threads(os.cpu_count() or 1)
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu, "dtype": a.dtype, "host_threads": torch.get_num_threads()}), flush=True)
    rows = []
    for case in a.cases.split(","):
        name, batch = case.split(":")
        eng = capi.Engine(CONFIGS[name], dt)
        eng.load_state_dict(synth_state_dict(CONFIGS[name], 1))
        eng.set_option("cuda_graph", 1)
        for src in a.sources.split(","):
            h, w = (int(v) for v in src.split("x"))
            r = measure(eng, name, int(batch), h, w, a.steps, a.warmup, a.rounds)
            r["gpu"] = gpu
            rows.append(r)
            print(json.dumps(r), flush=True)
        eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
