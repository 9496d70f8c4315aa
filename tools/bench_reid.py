"""Cost of tracking by appearance on the device (lwdetr_track_reid, LWDETR.track(appearance=True)) against tracking by
IoU alone (lwdetr_track_ex, LWDETR.track()).

    python tools/bench_reid.py [--frames 60] [--e2e-steps 10] [--rounds 3] [--configs small,xlarge] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_track_reid (D = 256, fp16 embeddings, as the decoder's rows) and lwdetr_track_ex (no motion) time per
           launch for 1, 32 and 256 streams, k = 300 entries per frame, on the scenes of tools/bench_track.py (20 and 150
           objects with seeded embeddings, and the 300-object crowd with random ones): a CUDA graph of `frames` launches
           over the pre-uploaded sequence, replayed from a reset tracker and timed by CUDA events; median and range of
           `rounds` replays, the two trackers alternating;
  e2e      LWDETR.track frames/s with and without appearance=True on 32 streams of 1080p NV12 (one frame each per call,
           fp16, CUDA graphs on, synthetic weights), host clock around `e2e-steps` calls, median and range of `rounds`
           alternating rounds.
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
from bench_track import K, crowd, spread  # noqa: E402
from models.lwdetr import LWDETR  # noqa: E402
import track_spec  # noqa: E402

D = 256


def sequences(streams, scene_name, frames):
    """Per frame: (scores [S, K], labels, boxes, embeddings fp16 [S, K, D]) on the device; at most 32 distinct streams,
    repeated beyond (the host generator is slow, and the kernel does the same work per stream)."""
    rng = np.random.default_rng(0)
    distinct = min(streams, 32)
    if scene_name == "crowd300":
        seqs = [crowd(frames, seed=s) for s in range(distinct)]
        embs = [[rng.normal(size=(K, D)).astype(np.float32) for _ in range(frames)] for _ in range(distinct)]
    else:
        objs = int(scene_name[5:])
        seqs, embs = [], []
        for s in range(distinct):
            f, _, _, e = track_spec.scene(1000 + s, frames, objects=objs, k=K, clutter=objs // 10, appearance=dict(seed=s, dim=D))
            seqs.append(f)
            embs.append(e)
    seqs = [seqs[s % distinct] for s in range(streams)]
    embs = [embs[s % distinct] for s in range(streams)]
    out = []
    for f in range(frames):
        out.append(tuple(torch.from_numpy(np.stack([seqs[s][f][i] for s in range(streams)])).cuda() for i in range(3))
                   + (torch.from_numpy(np.stack([embs[s][f] for s in range(streams)])).cuda().half(),))
    return out


def kernel_case(streams, scene_name, frames, rounds):
    seq = sequences(streams, scene_name, frames)
    ids = list(range(streams))
    runs = {}
    for name, tr, use in (("track_ex", capi.Tracker(streams, capacity=1024), False),
                          ("track_reid", capi.Tracker(streams, capacity=1024, embedding_dim=D), True)):
        call = (lambda f, tr=tr, use=use: tr.update(*seq[f][:3], ids, embeddings=seq[f][3] if use else None))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            call(0)                                      # warm-up (module load, smem attribute) outside the capture
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = [call(f) for f in range(frames)]
        runs[name] = (tr, graph, outs, [])
    for r in range(rounds + 1):
        for name, (tr, graph, _, per) in runs.items():
            tr.reset(ids)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            if r:                                        # the first replay is a warm-up
                per.append(e0.elapsed_time(e1) / frames)
    res = {"case": "kernel", "streams": streams, "scene": scene_name, "k": K, "dim": D, "frames": frames}
    for name, (tr, _, outs, per) in runs.items():
        res[name] = {"ms_per_launch": spread(per), "us_per_stream_frame": round(statistics.median(per) * 1000 / streams, 3),
                     "mean_output_tracks_per_frame": round(float(torch.stack([o[5] for o in outs]).float().mean()), 1)}
        tr.close()
    return res


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
    t_iou, t_app = capi.Tracker(n), capi.Tracker(n, embedding_dim=cfg.hidden_dim)
    iou = lambda i: models[0].track(dev(i), t_iou, colorspace="bt709")
    app = lambda i: models[1].track(dev(i), t_app, colorspace="bt709", appearance=True)

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    ri, ra = [], []
    for _ in range(rounds):
        for step, acc in ((iou, ri), (app, ra)):
            rate(step, 3)
            acc.append(rate(step, steps))
    for m in models:
        m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (h, w),
            "track_frames_per_s": spread(ri, 1), "track_appearance_frames_per_s": spread(ra, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reid.py needs a GPU")
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    for streams in (1, 32, 256):
        for scene_name in ("scene20", "scene150", "crowd300"):
            emit(kernel_case(streams, scene_name, a.frames, a.rounds))
    for name in a.configs.split(","):
        emit(e2e_case(name, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
