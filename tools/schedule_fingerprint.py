"""Fingerprint of the engine's forward schedule over the configurations, dtypes, input forms and options the planner
branches on: per case the op list (label, flops, bytes), the packed weight arena's size, and a sha256 of every output
tensor and of the requested debug captures.  Two builds that plan and compute the same forward write identical files, so
a host-side change to the planner can be checked by running this on both and comparing the JSON.
    python tools/schedule_fingerprint.py --out fingerprint.json [--cases tiny_f16_b2,...]
Uses only the public Python API (b200.capi.Engine).  Needs a CUDA device."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_images, synth_state_dict  # noqa: E402

DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16, "e4m3": torch.float8_e4m3fn}
CAPTURES = ("block0", "level0", "dec2")


def sha(t):
    t = t.detach().contiguous().cpu()
    return hashlib.sha256(t.view(torch.uint8).numpy().tobytes() if t.dtype != torch.bool else t.numpy().tobytes()).hexdigest()


def outputs(res):
    """sha256 of every tensor in a forward's result dict, by a flat name."""
    out = {"pred_logits": sha(res["pred_logits"]), "pred_boxes": sha(res["pred_boxes"])}
    for i, a in enumerate(res.get("aux_outputs", [])):
        out["aux%d_logits" % i], out["aux%d_boxes" % i] = sha(a["pred_logits"]), sha(a["pred_boxes"])
    if "enc_outputs" in res:
        out["enc_logits"], out["enc_boxes"] = sha(res["enc_outputs"]["pred_logits"]), sha(res["enc_outputs"]["pred_boxes"])
        out["topk_index"] = sha(res["topk_index"])
    return out


def entry(eng, res, captures=None):
    torch.cuda.synchronize()
    e = {"ops": [[lab, fl, by] for lab, fl, by in eng.ops()], "arena_bytes": eng.arena_bytes(), "outputs": outputs(res)}
    if captures:
        e["captures"] = {k: (sha(v) if v is not None else None) for k, v in eng.capture_results().items()}
    return e


def engine(name, dt):
    cfg = CONFIGS[name]
    eng = capi.Engine(cfg, DTYPES[dt])
    eng.load_state_dict(synth_state_dict(cfg, 1))
    return eng


def images(B, size, seed=0):
    return synth_images(B, seed, size).cuda()


def u8(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8).cuda()


def nv12(h, w, seed):
    rng = np.random.default_rng(seed)
    luma = rng.integers(0, 256, (h, w), dtype=np.uint8)
    chroma = rng.integers(0, 256, ((h + 1) // 2, 2 * ((w + 1) // 2)), dtype=np.uint8)
    return torch.from_numpy(luma).cuda(), torch.from_numpy(chroma).cuda()


def case_plain(name, dt, B, size=(640, 640), graph=False, fuse_ln=None):
    """B images at `size`: one eager forward, then (graph=True) with cuda_graph on - the capturing call and a replay."""
    def run():
        eng = engine(name, dt)
        if fuse_ln is not None:
            eng.set_option("fuse_layernorm", fuse_ln)
        x = images(B, size)
        r = {"eager": entry(eng, eng.forward(x))}
        if graph:
            eng.set_option("cuda_graph", 1)
            r["graph_capture"] = entry(eng, eng.forward(x))
            r["graph_replay"] = entry(eng, eng.forward(x))
        eng.close()
        return r
    return run


def case_captures():
    eng = engine("tiny", "f16")
    for lab in CAPTURES:
        eng.capture(lab, 1 << 24)
    r = entry(eng, eng.forward(images(2, (640, 640))), captures=True)
    eng.close()
    return r


def case_u8_mask():
    eng = engine("tiny", "f16")
    x = u8(2, 640, 640, 3)
    r = {"u8": entry(eng, eng.forward(x))}
    mask = torch.zeros(2, 640, 640, dtype=torch.bool)
    mask[0, :, 512:] = True
    mask[1, 448:, :] = True
    r["f32_mask"] = entry(eng, eng.forward(images(2, (640, 640)), mask=mask.cuda()))
    eng.close()
    return r


def case_frames():
    eng = engine("tiny", "f16")
    rgb = [u8(1, 480, 640, 10)[0], u8(1, 375, 501, 11)[0], u8(1, 1080, 1920, 12)[0]]
    kw = dict(fit="keep_aspect", short_side=512, max_side=704)
    r = {"rgb_keep_aspect": entry(eng, eng.forward_frames(rgb, **kw))}
    frames = [nv12(480, 640, 20), nv12(375, 501, 21), nv12(1080, 1920, 22)]
    r["nv12_keep_aspect"] = entry(eng, eng.forward_frames(frames, colorspace=["bt709", "bt709_full", "bt601"], **kw))
    r["nv12_stretch"] = entry(eng, eng.forward_frames(frames, colorspace="bt601"))
    eng.close()
    return r


def case_failed_plan():
    """A batch whose workspace would need a buffer past 2^31-1 elements fails inside the planner; the engine must then plan
    and compute the next forward exactly as a fresh engine does."""
    eng = engine("tiny", "f16")
    small = [u8(1, 8, 8, 30 + i)[0] for i in range(400)]
    try:
        eng.forward_frames(small, size=(1344, 1344), want_aux=False)
        err = None
    except RuntimeError as e:
        err = str(e)
    r = {"error": err, "ops_after_failure": len(eng.ops())}
    x = images(2, (640, 640))
    r["after"] = entry(eng, eng.forward(x))
    eng.close()
    fresh = engine("tiny", "f16")
    r["fresh_matches"] = entry(fresh, fresh.forward(x)) == r["after"]
    fresh.close()
    return r


def case_fuse_toggle():
    eng = engine("tiny", "f16")
    x = images(2, (640, 640))
    r = {}
    for step, v in enumerate((1, 0, 1)):
        eng.set_option("fuse_layernorm", v)
        r["step%d_fuse%d" % (step, v)] = entry(eng, eng.forward(x))
    eng.close()
    return r


def all_cases():
    cases = {}
    for name in ("tiny", "small", "medium", "large", "xlarge"):
        for dt in ("f16", "bf16"):
            cases["%s_%s_b2" % (name, dt)] = case_plain(name, dt, 2, graph=True)
    for name in ("tiny", "small"):
        for B in (1, 16):
            cases["%s_f16_b%d" % (name, B)] = case_plain(name, "f16", B)
    for name in ("tiny", "medium"):
        cases["%s_f16_nofuse" % name] = case_plain(name, "f16", 2, fuse_ln=0)
    for name in ("small", "xlarge"):
        cases["%s_e4m3_b2" % name] = case_plain(name, "e4m3", 2, graph=True)
    cases["small_f16_448x768"] = case_plain("small", "f16", 2, size=(448, 768))
    cases["large_f16_1024"] = case_plain("large", "f16", 2, size=(1024, 1024))
    cases["xlarge_f16_768x1344"] = case_plain("xlarge", "f16", 2, size=(768, 1344))
    cases["tiny_u8_mask"] = case_u8_mask
    cases["tiny_frames"] = case_frames
    cases["tiny_failed_plan"] = case_failed_plan
    cases["tiny_fuse_toggle"] = case_fuse_toggle
    cases["tiny_captures"] = case_captures
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--cases", default="", help="comma-separated case names (default: all)")
    a = ap.parse_args()
    cases = all_cases()
    names = [c for c in a.cases.split(",") if c] or list(cases)
    res = {}
    for n in names:
        res[n] = cases[n]()
        print(n, "done", flush=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
