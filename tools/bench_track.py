"""Rate of multi-object tracking on the device (lwdetr_track, LWDETR.track) and of the numpy specification on the host.

    python tools/bench_track.py [--frames 60] [--e2e-steps 10] [--rounds 3] [--configs small,xlarge] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_track time per launch for 1, 32 and 256 streams, k = nq = 300 entries per frame, synthetic scenes of 20 and
           150 objects (tools/track_spec.scene) and a crowd scene of 300 objects side by side whose first association is one
           component: a CUDA graph of `frames` launches (one frame of every stream each) over the pre-uploaded sequence is
           replayed from a reset tracker, timed by CUDA events; median and range of `rounds` replays;
  e2e      LWDETR.track frames/s against LWDETR.detect frames/s on the same 32 NV12 1080p frames (32 streams, one frame
           each per call, fp16, CUDA graphs on, synthetic weights), host clock around `e2e-steps` calls, alternating rounds;
  host     the numpy specification (tools/track_spec.py) per frame of one stream on the host, labelled as the reference
           point of a host tracker (it is not an optimised tracker).
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
import track_spec  # noqa: E402

K = 300


def spread(v, nd=4):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd)}


def crowd(frames, k=K, n=300, seed=0):
    rng = np.random.default_rng(seed)
    cx = 300 + np.arange(n) * 4.0
    out = []
    for f in range(frames):
        cx = cx + 1.0
        b = np.stack([cx - 30, 400 + rng.normal(0, 0.5, n), cx + 30, 520 + rng.normal(0, 0.5, n)], 1).astype(np.float32)
        out.append(track_spec.pad(rng.uniform(0.6, 0.95, n).astype(np.float32), np.zeros(n, np.int32), b, k))
    return out


def kernel_case(streams, scene_name, frames, rounds):
    if scene_name == "crowd300":
        seqs = [crowd(frames, seed=s) for s in range(streams)]
    else:
        objs = int(scene_name[5:])
        seqs = [track_spec.scene(1000 + s, frames, objects=objs, k=K, clutter=objs // 10) for s in range(streams)]
    sc = torch.from_numpy(np.stack([[seqs[s][f][0] for s in range(streams)] for f in range(frames)])).cuda()
    lb = torch.from_numpy(np.stack([[seqs[s][f][1] for s in range(streams)] for f in range(frames)])).cuda()
    bx = torch.from_numpy(np.stack([[seqs[s][f][2] for s in range(streams)] for f in range(frames)])).cuda()
    tr = capi.Tracker(streams, capacity=1024)
    ids = list(range(streams))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        tr.update(sc[0], lb[0], bx[0], ids)              # warm-up (module load, smem attribute) outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [tr.update(sc[f], lb[f], bx[f], ids) for f in range(frames)]
    per = []
    for r in range(rounds + 1):
        tr.reset(ids)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        if r:                                            # the first replay is a warm-up
            per.append(e0.elapsed_time(e1) / frames)
    tracks = float(torch.stack([o[5] for o in outs]).float().mean())
    tr.close()
    return {"case": "kernel", "streams": streams, "scene": scene_name, "k": K, "frames": frames,
            "ms_per_launch": spread(per), "us_per_stream_frame": round(statistics.median(per) * 1000 / streams, 3),
            "mean_output_tracks_per_frame": round(tracks, 1)}


def host_case(scene_name, frames):
    objs = int(scene_name[5:])
    seq = track_spec.scene(1000, frames, objects=objs, k=K, clutter=objs // 10)
    st = track_spec.Stream(track_spec.params(capacity=1024))
    t0 = time.perf_counter()
    for f in seq:
        st.update(*f)
    ms = (time.perf_counter() - t0) * 1000 / frames
    return {"case": "host_numpy_spec", "what": "tools/track_spec.py on the host CPU, one stream, not an optimised tracker",
            "scene": scene_name, "k": K, "frames": frames, "ms_per_frame": round(ms, 3)}


def e2e_case(name, steps, rounds):
    cfg = CONFIGS[name]
    models = []
    for _ in range(2):                                   # one engine each: the two paths keep their own plans
        m = LWDETR(cfg, compute_dtype=torch.float16).eval()
        m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
        m.cuda()
        m.engine().set_option("cuda_graph", 1)
        models.append(m)
    n, h, w = 32, 1080, 1920
    g = torch.Generator().manual_seed(1)
    host = [torch.randint(0, 256, (n, h * 3 // 2, w), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    tr = capi.Tracker(n)
    track = lambda i: models[0].track(dev(i), tr, colorspace="bt709")
    detect = lambda i: [d["scores"].shape for d in models[1].detect(dev(i), colorspace="bt709")]

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    rt, rd = [], []
    for _ in range(rounds):
        for step, acc in ((track, rt), (detect, rd)):
            rate(step, 3)
            acc.append(rate(step, steps))
    for m in models:
        m.engine().close()
    tr.close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (h, w),
            "track_frames_per_s": spread(rt, 1), "detect_frames_per_s": spread(rd, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track.py needs a GPU")
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    for streams in (1, 32, 256):
        for scene_name in ("scene20", "scene150", "crowd300"):
            emit(kernel_case(streams, scene_name, a.frames, a.rounds))
    for scene_name in ("scene20", "scene150"):
        emit(host_case(scene_name, a.frames))
    for name in a.configs.split(","):
        emit(e2e_case(name, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
