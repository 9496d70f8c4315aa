"""Tracking between detections on the device: what a flow frame costs against a detector frame.

  flow       lwdetr_track_flow (the flow kernels and the tracker step) per call, replayed from a CUDA graph, for 1 / 32 / 256
             streams of 1080p frames x 20 / 150 tracks at grid 10 (rendered sprites; tracks from true boxes);
  observe    lwdetr_gmc_observe against lwdetr_gmc_estimate per call, 32 streams of 1080p RGB, CUDA-graph replay;
  e2e        model.track() frames/s on 32 streams of 1080p NV12 (synthetic weights, noise frames) with detect_every 1 / 2 / 4
             at grid 10, and 4 at grid 4: median and range of alternating rounds, with the mean output tracks per keyframe
             and per flow frame of the warm-up calls.
Prints one JSON line per case.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "lw-detr_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402
from bench_resolution import gpu_info  # noqa: E402
from models.lwdetr import LWDETR  # noqa: E402


def spread(v, nd=4):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd), "n": len(v)}


def graph_ms(fn, reps=50):
    """ms per replay of a CUDA graph of fn (one warm-up call first)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def frames_1080p(n, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (1, 1080 // 8, 1920 // 8, 3), generator=g, dtype=torch.uint8)
    img = torch.nn.functional.interpolate(base.permute(0, 3, 1, 2).float(), size=(1080, 1920), mode="bilinear").round().byte()
    img = img.permute(0, 2, 3, 1).contiguous().cuda()
    return [torch.roll(img[0], shifts=(i % 7, 3 * (i % 5)), dims=(0, 1)).contiguous() for i in range(n)]


def flow_case(streams, tracks, rounds):
    est = capi.MotionEstimator(streams)
    flow = capi.BoxFlow(est)
    trk = capi.Tracker(streams, capacity=max(tracks + 8, 32))
    fr = frames_1080p(2, streams)
    rng = np.random.default_rng(tracks)
    x = rng.uniform(0, 1700, (streams, tracks))
    y = rng.uniform(0, 900, (streams, tracks))
    bx = torch.from_numpy(np.stack([x, y, x + 120, y + 160], 2).astype(np.float32)).cuda()
    ids = list(range(streams))
    est.observe([fr[0]] * streams, ids)
    trk.update(torch.full((streams, tracks), 0.9).cuda(), torch.zeros(streams, tracks, dtype=torch.int32).cuda(), bx, ids)
    est.observe([fr[1]] * streams, ids)
    res = []
    for _ in range(rounds):
        res.append(graph_ms(lambda: flow.propagate(trk, ids, max_out=tracks)))
    # each replay is one more flow frame on the same two pyramids: the tracks stay where the flow found them
    return {"case": "flow", "streams": streams, "tracks": tracks, "grid": int(flow.params.grid), "ms_per_call": spread(res, 4)}


def observe_case(rounds):
    n = 32
    fr = frames_1080p(n, 0)
    est = capi.MotionEstimator(n)
    fb = capi.Frames(fr, est.device)
    est.estimate(fb)
    ro, re = [], []
    for _ in range(rounds):
        ro.append(graph_ms(lambda: est.observe(fb)))
        re.append(graph_ms(lambda: est.estimate(fb)))
    return {"case": "observe_vs_estimate", "streams": n, "source": "1080x1920 rgb", "observe_ms": spread(ro, 4), "estimate_ms": spread(re, 4)}


def e2e_case(name, steps, rounds):
    cfg = CONFIGS[name]
    m = LWDETR(cfg, compute_dtype=torch.float16).eval()
    m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    m.cuda()
    m.engine().set_option("cuda_graph", 1)
    n, h, w = 32, 1080, 1920
    g = torch.Generator().manual_seed(1)
    host = [torch.randint(0, 256, (n, h * 3 // 2, w), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    runs = {}
    for every, grid in ((1, None), (2, 10), (4, 10), (4, 4)):
        tr = capi.Tracker(n)
        kw = {} if every == 1 else dict(detect_every=every, flow=capi.BoxFlow(capi.MotionEstimator(n), grid=grid))
        runs["detect_every_%d" % every + ("" if grid in (None, 10) else "_grid%d" % grid)] = (tr, kw)
    rates = {e: [] for e in runs}
    tracks = {e: [0, 0, 0, 0] for e in runs}          # output tracks and frames, on keyframes and on flow frames

    def rate(run, k, count=False):
        tr, kw = runs[run]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            out = m.track(dev(i), tr, colorspace="bt709", **kw)
            if count:
                for d in out:
                    flow = len(d["queries"]) > 0 and int(d["queries"][0]) < 0
                    tracks[run][2 * flow] += len(d["ids"])
                    tracks[run][2 * flow + 1] += 1
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    for _ in range(rounds):
        for run in runs:
            rate(run, 4, count=True)           # warm-up calls, whose track counts are reported
            rates[run].append(rate(run, steps))
    m.engine().close()
    per = {e: {"keyframes": round(v[0] / max(v[1], 1), 1), "flow_frames": round(v[2] / max(v[3], 1), 1)} for e, v in tracks.items()}
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (h, w),
            "track_frames_per_s": {e: spread(v, 1) for e, v in rates.items()}, "output_tracks_per_frame": per}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=8)
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flow.py needs a GPU")
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    for streams in (1, 32, 256):
        for tracks in (20, 150):
            emit(flow_case(streams, tracks, a.rounds))
    emit(observe_case(a.rounds))
    for name in a.configs.split(","):
        emit(e2e_case(name, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
