"""Rate of tiled detection (LWDETR.detect_tiled) against whole-frame detection (LWDETR.detect) on high-resolution frames.

    python tools/bench_tiled.py [--configs small,xlarge] [--sources 1080x1920:4,2160x3840:1] [--steps 10] [--warmup 3]
                                [--rounds 3] [--merge-iters 200] [--out FILE]

Per (config, source size, frames per call, RGB or NV12), pinned host uint8 frames (packed NV12 [3h/2, w], colorspace
"bt709", for NV12) are copied to the device and detected; the frame counts per call are chosen so that one call runs about
32 views at 640 x 640 (1080p: 4 frames x 9 views, 4K: 1 frame x 33 views; tile 640, overlap 0.2, per_view 100, fp16,
CUDA graphs on).  Reported, as the median and range of `rounds` alternating rounds of `steps` calls timed by a host clock:
  tiled   frames/s and views/s of detect_tiled (its per-frame count read-back included);
  whole   frames/s of detect() on the same frames (one 640 x 640 view per frame), on a second engine of the same weights
          (an engine keeps one plan; the two paths run different batch sizes).
Also, on the candidates of the real views: the merge kernel's own time (CUDA events around replays of a CUDA graph of 20
launches, so the Python call and its argument packing are not in it), the cost of one capi.tile_merge call from Python
(CUDA events around `merge-iters` back-to-back calls: argument packing, output allocation, launch), and, when torchvision's
CUDA ops are present, torchvision.ops.batched_nms called per frame on the same candidates (moved to frame pixels, IoU 0.5;
torchvision has no IoS; per call from Python, like merge_call_ms), else "not measured".  Synthetic weights: the rates do not depend
on the values, the candidate geometry does a little.  The GPU's name and power limit are read in the same run.  One JSON
line per case; --out also writes the list.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS, tile_views  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402
from bench_resolution import events_ms, gpu_info  # noqa: E402
from models.lwdetr import LWDETR, tile_crops  # noqa: E402

TILE, OVERLAP, PER_VIEW = 640, 0.2, 100


def host_rate(step, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(i)
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def spread(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)}


def merge_timing(model, frames, colorspace, iters):
    """(candidates per frame, merge kernel ms, merge ms per Python call, torchvision batched_nms ms per call or None) on the
    real views' output."""
    fb = capi.Frames(frames, colorspace=colorspace)
    (H, W), views = tile_views(model.cfg, fb.sizes, TILE, OVERLAP, True, None, PER_VIEW)
    out = model.engine().forward_frames(tile_crops(fb, views), size=(H, W), dsts=[(v[5], v[6]) for v in views], want_aux=False)
    sizes = torch.tensor([(v[3], v[4]) for v in views], dtype=torch.float32, device="cuda")
    s, l, b = capi.postprocess(out["pred_logits"], out["pred_boxes"], sizes, PER_VIEW)
    tv = [(v[0], v[2], v[1]) for v in views]
    F = len(fb.items)
    merge = lambda i: capi.tile_merge(s, l, b, tv, F, 0.0, 0.5, "ios", 300)
    merge(0)
    call_ms = events_ms(merge, iters) / iters
    # the kernel alone: `reps` launches captured in one CUDA graph (the host-side argument packing happens at capture), the
    # graph replayed; what remains beyond the kernel is the graph's per-node launch gap
    reps = 20
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            merge(0)
    graph.replay()
    kernel_ms = events_ms(lambda i: graph.replay(), max(iters // reps, 5)) / (max(iters // reps, 5) * reps)
    nms_ms = None
    try:
        import torchvision
        off = torch.tensor([[x0, y0, x0, y0] for _, x0, y0 in tv], dtype=torch.float32, device="cuda")
        fboxes = b + off[:, None, :]
        per_frame = []
        for f in range(F):
            idx = [i for i, v in enumerate(tv) if v[0] == f]
            per_frame.append((fboxes[idx].reshape(-1, 4), s[idx].reshape(-1), l[idx].reshape(-1)))

        def nms(i):
            for bb, ss, ll in per_frame:
                torchvision.ops.batched_nms(bb, ss, ll, 0.5)[:300]
        nms(0)
        nms_ms = events_ms(nms, max(iters // 10, 5)) / max(iters // 10, 5)
    except (ImportError, RuntimeError, NotImplementedError):
        nms_ms = None
    return len(views) // F * PER_VIEW, kernel_ms, call_ms, nms_ms


def measure(model, whole_model, h, w, n, nv12, steps, warmup, rounds, merge_iters):
    g = torch.Generator().manual_seed(h * 7 + w)
    shape = (n, h * 3 // 2, w) if nv12 else (n, h, w, 3)
    host = [torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    cs = "bt709" if nv12 else None
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    tiled = lambda i: model.detect_tiled(dev(i), tile=TILE, overlap=OVERLAP, per_view=PER_VIEW, colorspace=cs)
    whole = lambda i: [d["scores"].shape for d in whole_model.detect(dev(i), num_select=PER_VIEW, colorspace=cs)]
    nviews = len(tile_views(model.cfg, [(h, w)] * n, TILE, OVERLAP, True, None, PER_VIEW)[1])
    rt, rw = [], []
    for r in range(rounds):
        for step, acc in ((tiled, rt), (whole, rw)):
            host_rate(step, warmup)
            acc.append(host_rate(step, steps) * n)
    cand, kernel_ms, call_ms, nms_ms = merge_timing(model, dev(0), cs, merge_iters)
    return {"source": "%dx%d" % (h, w), "format": "nv12" if nv12 else "rgb", "frames_per_call": n, "views_per_call": nviews,
            "tiled_frames_per_s": spread(rt), "tiled_views_per_s": spread([x * nviews / n for x in rt]),
            "whole_frames_per_s": spread(rw), "candidates_per_frame": cand, "merge_kernel_ms": round(kernel_ms, 4),
            "merge_call_ms": round(call_ms, 4),
            "torchvision_batched_nms_ms": round(nms_ms, 4) if nms_ms is not None else "not measured"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--sources", default="1080x1920:4,2160x3840:1")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--merge-iters", type=int, default=200)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiled.py needs a GPU")
    info = gpu_info()
    res = []
    for name in a.configs.split(","):
        cfg = CONFIGS[name]
        models = []
        for _ in range(2):      # one engine each: an engine keeps one plan, and the two paths run different batch sizes
            m = LWDETR(cfg, compute_dtype=torch.float16).eval()
            m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
            m.cuda()
            m.engine().set_option("cuda_graph", 1)
            models.append(m)
        for src in a.sources.split(","):
            hw, n = src.split(":")
            h, w = (int(x) for x in hw.split("x"))
            for nv12 in (False, True):
                r = {"config": name, "dtype": "fp16", "gpu": info}
                r.update(measure(models[0], models[1], h, w, int(n), nv12, a.steps, a.warmup, a.rounds, a.merge_iters))
                print(json.dumps(r), flush=True)
                res.append(r)
        for m in models:
            m.engine().close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
