"""Cost of camera-motion estimation on the device (lwdetr_gmc_estimate, LWDETR.track(motion=...)) and of BoT-SORT's method
on the host.

    python tools/bench_gmc.py [--frames 6] [--rounds 3] [--e2e-steps 10] [--configs small,xlarge] [--cases estimator,host,e2e]
                              [--out FILE]

Reported, one JSON line per case, with the GPU's name, power limit and SM clocks read in the same run:
  estimator  lwdetr_gmc_estimate time per call for 1 and 32 streams at 720p, 1080p and 4K, RGB and NV12: a CUDA graph of
             `frames` calls (one frame of every stream each, textured frames shifted from call to call) over pre-uploaded
             frames is replayed, timed by CUDA events; median and range of `rounds` replays;
  host       tools/gmc_spec.botsort_gmc (BoT-SORT's sparseOptFlow with cv2) per frame on the host CPU, same frames, labelled
             as host time;
  e2e        LWDETR.track frames/s with and without motion= on the same 32 NV12 1080p frames (32 streams, one frame each per
             call, fp16, CUDA graphs on, synthetic weights), host clock around `e2e-steps` calls, alternating rounds; the
             frames are textured and shifted by a few pixels from call to call (a moving camera), or random noise (two
             unrelated frames: the estimator's worst case, every corner runs Lucas-Kanade to its iteration limit).
Needs a GPU."""
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
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_state_dict  # noqa: E402
from bench_resolution import gpu_info  # noqa: E402
from models.lwdetr import LWDETR  # noqa: E402
import gmc_spec  # noqa: E402

SIZES = {"720p": (720, 1280), "1080p": (1080, 1920), "4k": (2160, 3840)}


def spread(v, nd=4):
    return {"median": round(statistics.median(v), nd), "min": round(min(v), nd), "max": round(max(v), nd)}


def frames_for(res, streams, frames, fmt):
    """frames x streams device frames: one textured frame per resolution, shifted per stream and per call."""
    h, w = SIZES[res]
    base = torch.from_numpy(gmc_spec.textured_frame(h, h, w)).cuda()
    out = []
    for f in range(frames):
        row = []
        for s in range(streams):
            rgb = torch.roll(base, shifts=(3 * f + s, 5 * f + 2 * s), dims=(0, 1))
            if fmt == "rgb":
                row.append(rgb)
            else:
                luma = ((rgb[..., 0].int() * 66 + rgb[..., 1].int() * 129 + rgb[..., 2].int() * 25 + 128) >> 8) + 16
                row.append((luma.to(torch.uint8).contiguous(), torch.full((h // 2, w), 128, dtype=torch.uint8, device="cuda")))
        out.append(row)
    return out


def estimator_case(res, streams, fmt, frames, rounds):
    h, w = SIZES[res]
    seq = frames_for(res, streams, frames, fmt)
    est = capi.MotionEstimator(streams, max_height=h, max_width=w)
    ids = list(range(streams))
    cs = None if fmt == "rgb" else "bt709"
    batches = [capi.Frames(row, colorspace=cs) for row in seq]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        est.estimate(batches[0], ids)                     # warm-up (module load, smem attribute) outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = [est.estimate(b, ids) for b in batches]
    per = []
    for r in range(rounds + 1):
        est.reset(ids)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        if r:                                             # the first replay is a warm-up
            per.append(e0.elapsed_time(e1) / frames)
    ok = float(torch.stack([o[1] for o in outs[1:]]).eq(capi.GMC_OK).float().mean())
    inl = float(torch.stack([o[2] for o in outs[1:]]).float().mean())
    est.close()
    return {"case": "estimator", "source": "%s %s" % (res, fmt), "streams": streams, "calls": frames, "ms_per_call": spread(per),
            "ms_per_stream_frame": round(statistics.median(per) / streams, 4), "share_ok": round(ok, 3), "mean_inliers": round(inl, 1)}


def host_case(res, frames):
    seq = frames_for(res, 1, frames, "rgb")
    host = [row[0].cpu().numpy() for row in seq]
    t0 = time.perf_counter()
    for a, b in zip(host, host[1:]):
        gmc_spec.botsort_gmc(a, b)
    ms = (time.perf_counter() - t0) * 1000 / (len(host) - 1)
    return {"case": "host_botsort_gmc", "what": "BoT-SORT's sparseOptFlow with cv2 on the host CPU, one frame pair, host time",
            "source": "%s rgb" % res, "ms_per_frame": round(ms, 2)}


def e2e_case(name, source, steps, rounds):
    cfg = CONFIGS[name]
    m = LWDETR(cfg, compute_dtype=torch.float16).eval()
    m.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    m.cuda()
    m.engine().set_option("cuda_graph", 1)
    n, h, w = 32, 1080, 1920
    if source == "noise":                                # unrelated frames: every corner runs to the iteration limit
        g = torch.Generator().manual_seed(1)
        host = [torch.randint(0, 256, (n, h * 3 // 2, w), generator=g, dtype=torch.uint8).pin_memory() for _ in range(2)]
    else:                                                # textured frames, the camera shifting back and forth by (3, 5) px
        host = []
        for f in range(2):
            packed = torch.full((n, h * 3 // 2, w), 128, dtype=torch.uint8)
            for s, (y, _) in enumerate(frames_for("1080p", n, 2, "nv12")[f]):
                packed[s, :h] = y.cpu()
            host.append(packed.pin_memory())
    dev = lambda i: list(host[i & 1].cuda(non_blocking=True).unbind(0))
    t_plain, t_motion = capi.Tracker(n), capi.Tracker(n)
    est = capi.MotionEstimator(n, max_height=h, max_width=w)
    plain = lambda i: m.track(dev(i), t_plain, colorspace="bt709")
    moving = lambda i: m.track(dev(i), t_motion, colorspace="bt709", motion=est)

    def rate(step, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(k):
            step(i)
        torch.cuda.synchronize()
        return k * n / (time.perf_counter() - t0)
    rp, rm = [], []
    for _ in range(rounds):
        for step, acc in ((plain, rp), (moving, rm)):
            rate(step, 3)
            acc.append(rate(step, steps))
    m.engine().close()
    return {"case": "e2e", "config": name, "dtype": "fp16", "streams": n, "source": "%dx%d nv12 %s" % (h, w, source),
            "track_frames_per_s": spread(rp, 1), "track_with_motion_frames_per_s": spread(rm, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--configs", default="small,xlarge")
    ap.add_argument("--cases", default="estimator,host,e2e")
    ap.add_argument("--out")
    a = ap.parse_args()
    cases = a.cases.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gmc.py needs a GPU")
    info = gpu_info()
    res = []

    def emit(r):
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        res.append(r)
    for streams in (1, 32) if "estimator" in cases else ():
        for r in SIZES:
            for fmt in ("rgb", "nv12"):
                emit(estimator_case(r, streams, fmt, a.frames, a.rounds))
    for r in SIZES if "host" in cases else ():
        emit(host_case(r, a.frames))
    for name in a.configs.split(",") if "e2e" in cases else ():
        for source in ("textured", "noise"):
            emit(e2e_case(name, source, a.e2e_steps, a.rounds))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
