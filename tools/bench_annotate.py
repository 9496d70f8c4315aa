"""Cost of drawing into frames on the device (lwdetr_annotate / _nv12, LWDETR.track(annotate=)) and of the host way.

    python tools/bench_annotate.py [--rounds 3] [--host-frames 4] [--e2e-steps 10] [--skip kernel,host,e2e] [--out FILE]

Reported, one JSON line per case, with the GPU's name and power limit read in the same run:
  kernel   lwdetr_annotate time per call for 1 and 32 streams of 1080p and 4K, RGB and NV12 (bt709), 20 / 150 / 300 tracks per
           frame (boxes of 2-12 % of the frame side, labels with names, ids and scores), typical zones on every stream (4
           lines, 8 polygons of 16 vertices, occupancy text), privacy off and on (a third of the labels pixelated).  One call
           captured in a CUDA graph, 20 replays per timing, CUDA events; median of `rounds` timings.  GB/s counts the
           bytes of the 64 x 64 tiles that some primitive touches (read and written once each), from the tile cover of the
           same primitives (tools/annotate_spec.py), over the call's time;
  host     the host way: per frame, read back, cv2.cvtColor NV12 -> BGR, cv2.rectangle / cv2.putText per box, cvtColor back
           (BGR -> YUV I420, repacked to NV12) and upload; host clock per frame.  Not the same work as the kernel's (no zones,
           pixelation or label backgrounds; 4 colours; OpenCV's Hershey font at another size): an order of magnitude only;
  e2e      LWDETR.track frames/s with and without annotate= (zones on both) on 32 NV12 1080p frames (32 streams, fp16, CUDA
           graphs on, synthetic weights), host clock around `e2e-steps` calls, alternating rounds.
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

NAMES = ["person", "bicycle", "car", "motorcycle", "bus", "truck"]
SIZES = {"1080p": (1080, 1920), "4k": (2160, 3840)}


def spread(v, nd=4):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd)}


def scene(streams, n, h, w, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.uniform(0, 1, (streams, n, 2)) * (w, h)
    s = rng.uniform(0.02, 0.12, (streams, n, 2)) * (w, h)
    boxes = np.concatenate([c - s / 2, c + s / 2], -1).astype(np.float32)
    scores = rng.uniform(0.3, 1, (streams, n)).astype(np.float32)
    labels = rng.integers(0, len(NAMES), (streams, n)).astype(np.int32)
    ids = np.arange(1, n + 1, dtype=np.int32)[None].repeat(streams, 0)
    return scores, labels, boxes, ids


def touched_tiles(h, w, boxes, geo, scale):
    """Tiles of 64 x 64 that a box, its label or a zone's bounding box meets (an estimate of the bytes the draw kernel moves)."""
    ty, tx = (h + 63) // 64, (w + 63) // 64
    m = np.zeros((ty, tx), bool)

    def mark(x0, y0, x1, y1):
        x0, y0 = max(int(x0), 0), max(int(y0), 0)
        x1, y1 = min(int(np.ceil(x1)), w), min(int(np.ceil(y1)), h)
        if x1 > x0 and y1 > y0:
            m[y0 // 64:(y1 - 1) // 64 + 1, x0 // 64:(x1 - 1) // 64 + 1] = True
    for b in boxes:
        mark(*b)
        mark(b[0], b[1] - 8 * scale, b[0] + 6 * scale * 20, b[1])
    lines, polys = geo
    for l in lines:
        mark(min(l[0], l[2]) - 2, min(l[1], l[3]) - 2, max(l[0], l[2]) + 2, max(l[1], l[3]) + 2)
    for p in polys:
        p = np.asarray(p)
        mark(p[:, 0].min(), p[:, 1].min(), p[:, 0].max() + 1, p[:, 1].max() + 1)
    return int(m.sum())


def kernel_case(streams, size, fmt, n, privacy, rounds):
    h, w = SIZES[size]
    dev = "cuda"
    if fmt == "nv12":
        frames = [(torch.randint(0, 256, (h, w), dtype=torch.uint8, device=dev), torch.randint(0, 256, (h // 2, w), dtype=torch.uint8, device=dev))
                  for _ in range(streams)]
    else:
        frames = list(torch.randint(0, 256, (streams, h, w, 3), dtype=torch.uint8, device=dev).unbind(0))
    fb = capi.Frames(frames, colorspace="bt709" if fmt == "nv12" else None)
    sc, lab, bx, ids = (torch.from_numpy(x).to(dev) for x in scene(streams, n, h, w))
    z = capi.Zones(streams, num_classes=len(NAMES))
    geos = []
    for s in range(streams):
        geos.append(zone_spec.layout(s, size=(h, w), lines=4, polygons=8, vertices=16))
        z.set(s, *geos[-1])
    counts = torch.full((streams,), n, dtype=torch.int32, device=dev)
    _, occ, _, _ = z.update(ids, lab, bx, counts)
    ann = capi.Annotator(len(NAMES), names=NAMES, privacy=[1, 4] if privacy else ())
    call = lambda: ann.annotate(fb, sc, lab, bx, ids=ids, counts=counts, zones=z, occupancy=occ)  # noqa: E731
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    g.replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            g.replay()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1) / 20)
    bxh = bx.cpu().numpy()
    px = 3 if fmt == "rgb" else 1.5
    tiles = sum(touched_tiles(h, w, bxh[s], geos[s], 2) for s in range(streams))
    med = statistics.median(ms)
    return {"case": "kernel", "streams": streams, "size": size, "format": fmt, "tracks": n, "privacy": privacy,
            "ms_per_call": spread(ms), "touched_tiles": tiles, "touched_GB_per_s": round(2 * tiles * 4096 * px / (med * 1e-3) / 1e9, 1)}


def host_case(size, n, frames):
    import cv2
    h, w = SIZES[size]
    luma = torch.randint(0, 256, (h * 3 // 2, w), dtype=torch.uint8, device="cuda")
    sc, lab, bx, ids = scene(1, n, h, w)
    pal = capi_palette()
    t = []
    for _ in range(frames):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        img = cv2.cvtColor(luma.cpu().numpy(), cv2.COLOR_YUV2BGR_NV12)
        for j in range(n):
            x0, y0, x1, y1 = (int(v) for v in bx[0, j])
            c = pal[ids[0, j] % len(pal)]
            cv2.rectangle(img, (x0, y0), (x1, y1), c, 2)
            cv2.putText(img, "%s #%d %.2f" % (NAMES[lab[0, j]], ids[0, j], sc[0, j]), (x0, max(y0 - 4, 10)), cv2.FONT_HERSHEY_SIMPLEX, 0.5, c, 1)
        i420 = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)
        uv = np.stack([i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)], -1).reshape(h // 2, w)
        luma.copy_(torch.from_numpy(np.concatenate([i420[:h], uv])).cuda())
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return {"case": "host", "size": size, "format": "nv12", "tracks": n, "ms_per_frame": spread(t[1:] if len(t) > 1 else t, 2)}


def capi_palette():
    return [tuple(int(v) for v in c) for c in [(230, 25, 75), (60, 180, 75), (255, 225, 25), (0, 130, 200)]]


def e2e_case(name, steps, rounds):
    cfg = CONFIGS[name]
    m = LWDETR(cfg, compute_dtype=torch.float16).eval()
    m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    m.cuda()
    m.engine().set_option("cuda_graph", 1)
    n, (H, W) = 32, SIZES["1080p"]
    g = torch.Generator().manual_seed(1)
    host = [torch.randint(0, 256, (n, H * 3 // 2, W), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))  # noqa: E731
    ta, tb = capi.Tracker(n), capi.Tracker(n)
    za, zb = capi.Zones(n, num_classes=cfg.num_classes), capi.Zones(n, num_classes=cfg.num_classes)
    for s in range(n):
        geo = zone_spec.layout(s, lines=4, polygons=8, vertices=16)
        za.set(s, *geo)
        zb.set(s, *geo)
    ann = capi.Annotator(cfg.num_classes)
    drawn = lambda i: m.track(dev(i), ta, colorspace="bt709", zones=za, annotate=ann)  # noqa: E731
    plain = lambda i: m.track(dev(i), tb, colorspace="bt709", zones=zb)  # noqa: E731

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    ry, rn = [], []
    for _ in range(rounds):
        for step, acc in ((drawn, ry), (plain, rn)):
            rate(step, 3)
            acc.append(rate(step, steps))
    m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12" % (H, W),
            "track_zones_frames_per_s": spread(rn, 1), "track_zones_annotate_frames_per_s": spread(ry, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-frames", type=int, default=4)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small")
    ap.add_argument("--skip", default="", help="comma-separated cases to leave out: kernel, host, e2e")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_annotate.py needs a GPU")
    skip = set(filter(None, a.skip.split(",")))
    gpu = gpu_info()
    out = open(a.out, "w") if a.out else None

    def emit(r):
        r["gpu"] = gpu
        line = json.dumps(r)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
    if "kernel" not in skip:
        for streams in (1, 32):
            for size in SIZES:
                for fmt in ("rgb", "nv12"):
                    for n in (20, 150, 300):
                        for privacy in (False, True):
                            emit(kernel_case(streams, size, fmt, n, privacy, a.rounds))
    if "host" not in skip:
        for size in SIZES:
            for n in (20, 150, 300):
                emit(host_case(size, n, a.host_frames))
    if "e2e" not in skip:
        for name in a.configs.split(","):
            emit(e2e_case(name, a.e2e_steps, a.rounds))


if __name__ == "__main__":
    main()
