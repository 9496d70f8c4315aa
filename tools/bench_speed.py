"""Cost of speed estimation on the device (lwdetr_speed_update, LWDETR.track(speed=)) and of the host way.

    python tools/bench_speed.py [--frames 30] [--host-frames 5] [--e2e-steps 10] [--rounds 3] [--configs small] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_speed_update time per launch for 1, 32 and 256 streams x 20, 150 and 300 tracks per stream (max_out 300)
           x window 30 and 64 (min_samples = window / 2).  Tracks are tracker-shaped outputs (stable ids, boxes moving across
           a 1080p frame); every stream has a camera homography.  The object is warmed up over `window` frames first, so
           every ring is full and every fit runs over the whole window; then a CUDA graph of `frames` launches is replayed,
           timed by CUDA events; median and range of `rounds` replays;
  host     the host way: per stream and frame, the tracker's outputs read back and the numpy restatement
           (tools/speed_spec.py) run on them; host clock per frame of all streams;
  e2e      LWDETR.track frames/s with and without speed= on the same 32 NV12 1080p frames (32 streams, one frame each per
           call, fp16, CUDA graphs on, synthetic weights), host clock around `e2e-steps` calls, alternating rounds.
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
from bench_zones import H, W, spread, tracks  # noqa: E402
from models.lwdetr import LWDETR  # noqa: E402
import speed_spec  # noqa: E402

HOMOGRAPHY = speed_spec.camera()["H"]


def drop_labels(seq):
    return [(ids, boxes, counts) for ids, _, boxes, counts in seq]


def kernel_case(streams, n, window, frames, rounds):
    seq = drop_labels(tracks(streams, n, window + frames, seed=streams * 1000 + n))
    e = capi.SpeedEstimator(streams, window=window, min_samples=window // 2)
    for s in range(streams):
        e.set(s, HOMOGRAPHY)
    ids = list(range(streams))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for f in range(window):                          # fills every ring; loads the module outside the capture
            e.update(*seq[f], ids)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [e.update(*seq[window + f], ids) for f in range(frames)]
    per = []
    for r in range(rounds + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        if r:                                            # the first replay is a warm-up
            per.append(e0.elapsed_time(e1) / frames)
    full = float((outs[-1][1][:, :n] == window).float().mean())
    e.close()
    return {"case": "kernel", "streams": streams, "tracks": n, "window": window, "frames": frames, "ms_per_launch": spread(per),
            "us_per_stream_frame": round(statistics.median(per) * 1000 / streams, 3), "full_window_share": round(full, 3)}


def host_case(streams, n, frames):
    seq = drop_labels(tracks(streams, n, 30 + frames, seed=streams * 1000 + n))
    st = [speed_spec.Stream(speed_spec.params()) for _ in range(streams)]
    for s in range(streams):
        st[s].set(HOMOGRAPHY)
    for ids, boxes, counts in seq[:30]:                 # full rings, untimed
        ids, boxes, counts = (t.cpu().numpy() for t in (ids, boxes, counts))
        for s in range(streams):
            st[s].update(ids[s], boxes[s], counts[s])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for ids, boxes, counts in seq[30:]:
        ids, boxes, counts = (t.cpu().numpy() for t in (ids, boxes, counts))
        for s in range(streams):
            st[s].update(ids[s], boxes[s], counts[s])
    ms = (time.perf_counter() - t0) * 1000 / frames
    return {"case": "host", "what": "read-back + tools/speed_spec.py per stream on the host CPU", "streams": streams, "tracks": n,
            "window": 30, "frames": frames, "ms_per_frame": round(ms, 3)}


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
    e = capi.SpeedEstimator(n)
    for s in range(n):
        e.set(s, HOMOGRAPHY)
    found = []
    with_speed = lambda i: found.append(sum(len(d["ids"]) for d in m.track(dev(i), ta, colorspace="bt709", speed=e)))
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
        for step, acc in ((with_speed, ry), (without, rn)):
            rate(step, 3)
            acc.append(rate(step, steps))
    m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (H, W),
            "track_frames_per_s": spread(rn, 1), "track_with_speed_frames_per_s": spread(ry, 1),
            "mean_tracks_per_frame": round(sum(found) / max(len(found), 1) / n, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--host-frames", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small")
    ap.add_argument("--skip", default="", help="comma-separated cases to leave out: kernel, host, e2e")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_speed.py needs a GPU")
    skip = set(filter(None, a.skip.split(",")))
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    if "kernel" not in skip:
        for window in (30, 64):
            for streams in (1, 32, 256):
                for n in (20, 150, 300):
                    emit(kernel_case(streams, n, window, a.frames, a.rounds))
    if "host" not in skip:
        for streams in (1, 32):
            for n in (20, 150, 300):
                emit(host_case(streams, n, a.host_frames))
    if "e2e" not in skip:
        for name in a.configs.split(","):
            emit(e2e_case(name, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
