"""Cost of line crossings and zone occupancy on the device (lwdetr_zones_update, LWDETR.track(zones=)) and of the host way.

    python tools/bench_zones.py [--frames 30] [--host-frames 10] [--e2e-steps 10] [--rounds 3] [--configs small,xlarge] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_zones_update time per launch for 1, 32 and 256 streams x 20, 150 and 300 tracks per stream (max_out 300)
           x two geometries per stream: "typical" (4 lines, 8 polygons of 16 vertices) and "limits" (32 lines, 32 polygons
           of 64 vertices: 2048).  Tracks are tracker-shaped outputs (stable ids, boxes moving across a 1080p frame and
           wrapping round, so lines are crossed and zones entered and left).  A CUDA graph of `frames` launches over the
           pre-uploaded sequence is replayed from a reset object, timed by CUDA events; median and range of `rounds` replays;
  host     the host way, as supervision's LineZone / PolygonZone run it: per stream and frame, the tracker's outputs read
           back and the numpy restatement (tools/zone_spec.py: vectorised geometry, a Python loop per track for the state)
           run on them; host clock per frame of all streams;
  e2e      LWDETR.track frames/s with and without zones= (typical geometry on every stream) on the same 32 NV12 1080p frames
           (32 streams, one frame each per call, fp16, CUDA graphs on, synthetic weights), host clock around `e2e-steps`
           calls, alternating rounds.
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
import zone_spec  # noqa: E402

MAX_OUT = 300
H, W = 1080, 1920


def spread(v, nd=4):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd)}


def geometry(name, seed):
    if name == "typical":
        return zone_spec.layout(seed, lines=4, polygons=8, vertices=16)
    return zone_spec.layout(seed, lines=32, polygons=32, vertices=64)


def tracks(streams, n, frames, seed=0):
    """Tracker-shaped outputs [frames] of (ids, labels, boxes, counts) for `streams` streams of n tracks (CUDA)."""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(0, W, (streams, n))
    cy = rng.uniform(0, H, (streams, n))
    vx = rng.normal(0, 12, (streams, n))
    vy = rng.normal(0, 6, (streams, n))
    hh = rng.uniform(40, 160, (streams, n))
    ww = hh * rng.uniform(0.3, 1.0, (streams, n))
    ids = np.zeros((streams, MAX_OUT), np.int32)
    ids[:, :n] = np.arange(1, n + 1)
    labels = np.zeros((streams, MAX_OUT), np.int32)
    labels[:, :n] = rng.integers(0, 3, (streams, n))
    out = []
    for _ in range(frames):
        cx = (cx + vx) % W
        cy = (cy + vy) % H
        b = np.zeros((streams, MAX_OUT, 4), np.float32)
        b[:, :n] = np.stack([cx - ww / 2, cy - hh / 2, cx + ww / 2, cy + hh / 2], -1)
        out.append(tuple(torch.from_numpy(x).cuda() for x in (ids, labels, b, np.full(streams, n, np.int32))))
    return out


def kernel_case(streams, n, geo, frames, rounds):
    seq = tracks(streams, n, frames, seed=streams * 1000 + n)
    z = capi.Zones(streams)
    for s in range(streams):
        z.set(s, *geometry(geo, s))
    ids = list(range(streams))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        z.update(*seq[0], ids)                           # warm-up (module load, smem attribute) outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [z.update(*seq[f], ids) for f in range(frames)]
    per = []
    for r in range(rounds + 1):
        z.reset(ids)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        if r:                                            # the first replay is a warm-up
            per.append(e0.elapsed_time(e1) / frames)
    events = float(torch.stack([o[3] for o in outs]).float().mean())
    z.close()
    return {"case": "kernel", "streams": streams, "tracks": n, "geometry": geo, "frames": frames, "ms_per_launch": spread(per),
            "us_per_stream_frame": round(statistics.median(per) * 1000 / streams, 3), "mean_events_per_stream_frame": round(events, 1)}


def host_case(streams, n, geo, frames):
    seq = tracks(streams, n, frames, seed=streams * 1000 + n)
    st = [zone_spec.Stream(zone_spec.params()) for _ in range(streams)]
    for s in range(streams):
        st[s].set(*geometry(geo, s))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for ids, labels, boxes, counts in seq:
        ids, labels, boxes, counts = (t.cpu().numpy() for t in (ids, labels, boxes, counts))
        for s in range(streams):
            st[s].update(ids[s], labels[s], boxes[s], counts[s])
    ms = (time.perf_counter() - t0) * 1000 / frames
    return {"case": "host", "what": "read-back + tools/zone_spec.py per stream on the host CPU", "streams": streams, "tracks": n,
            "geometry": geo, "frames": frames, "ms_per_frame": round(ms, 3)}


def e2e_case(name, steps, rounds):
    cfg = CONFIGS[name]
    m = LWDETR(cfg, compute_dtype=torch.float16).eval()
    m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    m.cuda()
    m.engine().set_option("cuda_graph", 1)
    n = 32
    g = torch.Generator().manual_seed(1)
    host = [torch.randint(0, 256, (n, H * 3 // 2, W), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    ta, tb = capi.Tracker(n), capi.Tracker(n)
    z = capi.Zones(n, num_classes=cfg.num_classes)
    for s in range(n):
        z.set(s, *geometry("typical", s))
    found = []
    with_zones = lambda i: found.append(sum(len(d["ids"]) for d in m.track(dev(i), ta, colorspace="bt709", zones=z)))
    without = lambda i: m.track(dev(i), tb, colorspace="bt709")

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    ry, rn = [], []
    for _ in range(rounds):
        for step, acc in ((with_zones, ry), (without, rn)):
            rate(step, 3)
            acc.append(rate(step, steps))
    m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (H, W),
            "track_frames_per_s": spread(rn, 1), "track_with_zones_frames_per_s": spread(ry, 1),
            "mean_tracks_per_frame": round(sum(found) / max(len(found), 1) / n, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--host-frames", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--skip", default="", help="comma-separated cases to leave out: kernel, host, e2e")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_zones.py needs a GPU")
    skip = set(filter(None, a.skip.split(",")))
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    if "kernel" not in skip:
        for geo in ("typical", "limits"):
            for streams in (1, 32, 256):
                for n in (20, 150, 300):
                    emit(kernel_case(streams, n, geo, a.frames, a.rounds))
    if "host" not in skip:
        for geo, streams in (("typical", 1), ("typical", 32), ("limits", 1)):
            for n in (20, 150, 300):
                emit(host_case(streams, n, geo, a.host_frames))
    if "e2e" not in skip:
        for name in a.configs.split(","):
            emit(e2e_case(name, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
