"""Cost of detection crops on the device (lwdetr_crops / _nv12, LWDETR.track(reid=)) against BoT-SORT's host way.

    python tools/bench_crops.py [--per-frame 16,64,300] [--iters 20] [--rounds 3] [--e2e-steps 10] [--configs small] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_crops on 32 frames of 1080p (RGB and NV12), 16 / 64 / 300 seeded boxes per frame (pedestrian-like, 20-300
           px wide, 40-600 px tall) to 256 x 128 fp16, both filters: a CUDA graph of `iters` launches timed by CUDA events,
           median and range of `rounds` replays.  GB/s of compulsory bytes (each crop's footprint read once: 3 bytes per pixel
           RGB, 1.5 NV12; the output written once; boxes and indices) over that time, and its share of the H100 SXM data
           sheet's 3.35 TB/s, which is a ceiling, not a reachable rate;
  host     BoT-SORT's way on the same boxes (RGB frames): the frames copied to the host, a Python loop of per-box slicing and
           cv2.resize(INTER_LINEAR), then the crops stacked and copied back (as float32 levels); NV12 frames also take
           cv2.cvtColor per frame; host clock around one whole pass after a synchronise;
  e2e      LWDETR.track frames/s on 32 streams of 1080p NV12 (fp16, CUDA graphs on, synthetic weights): IoU only,
           appearance=True, and reid= a stand-in CNN at random init (fp16) at 256 x 128; the tracker's track_thresh is set
           by the bench to the score quantile that keeps about `e2e-crops` entries per frame on these frames, so the crop
           count does not depend on what the synthetic weights score.
Needs a GPU."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402
from bench_resolution import gpu_info  # noqa: E402
from models.lwdetr import LWDETR  # noqa: E402

N_FRAMES, H, W, OUT = 32, 1080, 1920, (256, 128)
HBM_PEAK = 3.35e12


def spread(v, nd=3):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd)}


def frames(nv12, seed=1):
    g = torch.Generator().manual_seed(seed)
    if nv12:
        return capi.Frames(list(torch.randint(0, 256, (N_FRAMES, H * 3 // 2, W), generator=g, dtype=torch.uint8).cuda().unbind(0)),
                           colorspace="bt709")
    return capi.Frames(list(torch.randint(0, 256, (N_FRAMES, H, W, 3), generator=g, dtype=torch.uint8).cuda().unbind(0)))


def boxes(per_frame, seed=2):
    rng = np.random.default_rng(seed + per_frame)
    n = N_FRAMES * per_frame
    w, h = rng.uniform(20, 300, n), rng.uniform(40, 600, n)
    x, y = rng.uniform(0, W - w), rng.uniform(0, H - h)
    b = np.stack([x, y, x + w, y + h], 1).astype(np.float32)
    return b, np.repeat(np.arange(N_FRAMES, dtype=np.int32), per_frame)


def compulsory_bytes(b, nv12):
    x0, y0, x1, y1 = (np.clip(np.floor(b[:, i]), 0, s) for i, s in zip(range(4), (W, H, W, H)))
    px = ((x1 - x0) * (y1 - y0)).sum()
    return px * (1.5 if nv12 else 3) + len(b) * (3 * OUT[0] * OUT[1] * 2 + 16 + 4 + 1)


def kernel_case(nv12, per_frame, filter, iters, rounds):
    fb = frames(nv12)
    b, f = boxes(per_frame)
    bt, ft = torch.from_numpy(b).cuda(), torch.from_numpy(f).cuda()
    out = torch.empty(len(b), 3, *OUT, device="cuda", dtype=torch.float16)
    val = torch.empty(len(b), device="cuda", dtype=torch.int8)
    call = lambda: capi.crops(fb, bt, ft, OUT, filter, dtype=torch.float16, out=out, valid=val)
    call()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            call()
    g.replay()
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    ms = statistics.median(times)
    by = float(compulsory_bytes(b, nv12))
    return {"case": "kernel", "source": "%dx%d %s" % (H, W, "nv12" if nv12 else "rgb"), "frames": N_FRAMES, "crops_per_frame": per_frame,
            "filter": filter, "out": "%dx%d fp16" % OUT, "ms": spread(times, 4), "compulsory_MB": round(by / 1e6, 2),
            "GB_per_s": round(by / ms / 1e6, 1), "share_of_3.35TBps_ceiling": round(by / ms / 1e-3 / HBM_PEAK, 3)}


def host_case(nv12, per_frame):
    import cv2
    fb = frames(nv12)
    b, f = boxes(per_frame)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if nv12:
        host = [cv2.cvtColor(torch.cat([y.reshape(-1), c.reshape(-1)]).cpu().numpy().reshape(H * 3 // 2, W), cv2.COLOR_YUV2RGB_NV12)
                for y, c in fb.items]
    else:
        host = [x.cpu().numpy() for x in fb.items]
    crops = []
    for (x0, y0, x1, y1), fi in zip(b.astype(int), f):
        crops.append(cv2.resize(host[fi][y0:y1, x0:x1], (OUT[1], OUT[0]), interpolation=cv2.INTER_LINEAR))
    t = torch.from_numpy(np.stack(crops)).cuda().permute(0, 3, 1, 2).float()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    assert t.shape[0] == len(b)
    return {"case": "host", "source": "%dx%d %s" % (H, W, "nv12" if nv12 else "rgb"), "frames": N_FRAMES, "crops_per_frame": per_frame,
            "ms": round(ms, 2)}


class StandIn(torch.nn.Module):
    """A ReID-shaped CNN at random init (strided convolutions, global pooling, 512-wide embedding), fp16."""

    def __init__(self, D=512):
        super().__init__()
        c = [3, 32, 64, 128, 256]
        layers = []
        for a, b in zip(c[:-1], c[1:]):
            layers += [torch.nn.Conv2d(a, b, 3, stride=2, padding=1), torch.nn.ReLU()]
        self.net = torch.nn.Sequential(*layers, torch.nn.AdaptiveAvgPool2d(1), torch.nn.Flatten(), torch.nn.Linear(c[-1], D))

    def forward(self, x):
        return self.net(x.half()).float()


def e2e_case(name, steps, rounds, crops_per_frame):
    cfg = CONFIGS[name]
    models = []
    for _ in range(3):                                   # one engine each: the paths keep their own plans
        m = LWDETR(cfg, compute_dtype=torch.float16).eval()
        m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
        m.cuda()
        m.engine().set_option("cuda_graph", 1)
        models.append(m)
    n = N_FRAMES
    g = torch.Generator().manual_seed(1)
    host = [torch.randint(0, 256, (n, H * 3 // 2, W), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    out = models[2].engine().forward_frames(dev(0), colorspace="bt709", want_aux=False)
    sizes = torch.tensor([(H, W)] * n, dtype=torch.float32, device="cuda")
    sc = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)[0]
    thr = float(torch.quantile(sc.flatten().float(), 1.0 - crops_per_frame / cfg.num_queries))
    net = StandIn().cuda().half().eval()
    tp = dict(track_thresh=thr, new_track_thresh=min(1.0, thr + 0.1))
    t_iou, t_app = capi.Tracker(n, **tp), capi.Tracker(n, embedding_dim=cfg.hidden_dim, **tp)
    t_reid = capi.Tracker(n, embedding_dim=512, **tp)
    iou = lambda i: models[0].track(dev(i), t_iou, colorspace="bt709")
    app = lambda i: models[1].track(dev(i), t_app, colorspace="bt709", appearance=True)
    reid = lambda i: models[2].track(dev(i), t_reid, colorspace="bt709", reid=net)
    counts = []
    for i in range(2):
        o = models[2].engine().forward_frames(dev(i), colorspace="bt709", want_aux=False)
        s, _, b = capi.query_best(o["pred_logits"], o["pred_boxes"], sizes)
        counts.append(int(capi.crop_select(s, b, [(H, W)] * n, thr)[3].item()))

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    acc = {"iou": [], "appearance": [], "reid": []}
    for _ in range(rounds):
        for key, step in (("iou", iou), ("appearance", app), ("reid", reid)):
            rate(step, 3)
            acc[key].append(rate(step, steps))
    for m in models:
        m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (H, W),
            "crops_per_call": counts, "reid_net": "stand-in CNN, 4 strided 3x3 convs, D=512, fp16, 256x128 crops",
            "track_frames_per_s": spread(acc["iou"], 1), "track_appearance_frames_per_s": spread(acc["appearance"], 1),
            "track_reid_frames_per_s": spread(acc["reid"], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-frame", default="16,64,300")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--e2e-crops", type=int, default=16)
    ap.add_argument("--configs", default="small")
    ap.add_argument("--skip-host", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_crops.py needs a GPU")
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    per = [int(x) for x in a.per_frame.split(",")]
    for nv12 in (False, True):
        for p in per:
            for filt in ("bilinear", "antialias"):
                emit(kernel_case(nv12, p, filt, a.iters, a.rounds))
            if not a.skip_host:
                emit(host_case(nv12, p))
    for name in [c for c in a.configs.split(",") if c]:
        emit(e2e_case(name, a.e2e_steps, a.rounds, a.e2e_crops))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
