"""Generate tests/golden/*.npz by running the UNMODIFIED reference (imported via tools/ref_import.py from the
checkout named by $LWDETR_REFERENCE_SRC or staged under oracle/_ref) on the deterministic synthetic weights/inputs of
b200/synth.py.

    python tools/make_goldens.py [--postprocess-only | --padded-only | --seed5-only | --resolution-only]
Each fixture holds the reference's final outputs and strided samples of its intermediates (captured
with forward hooks), plus the state_dict names/shapes (tests/golden/state_dict_<cfg>.json).
"""
import dataclasses
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))

import ref_import  # noqa: E402
from b200.config import CONFIGS  # noqa: E402
from b200.synth import synth_images, synth_state_dict  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CASES = [("tiny", 2), ("small", 1), ("medium", 1), ("large", 1), ("xlarge", 1)]
WEIGHT_SEED, IMAGE_SEED = 1, 0


def sample(t, n=2048):
    f = t.detach().reshape(-1).float()
    step = max(1, f.numel() // n)
    return f[::step][:n].numpy().copy()


POST_SIZES = [[480.0, 640.0], [640.0, 427.0]]     # (height, width) per image, as PostProcess takes them


def make_postprocess_goldens():
    """Reference PostProcess.forward (lwdetr.py:515-544) on the reference's own golden predictions: pins the oracle's
    postprocess() and, through it, the fused device kernel.  Only needs the existing ref_<cfg>.npz fixtures."""
    rec = {}
    for name, B in CASES:
        cfg = CONFIGS[name]
        _, _, post = ref_import.build_reference(cfg)
        gold = np.load(os.path.join(GOLD, "ref_%s.npz" % name))
        out = {"pred_logits": torch.from_numpy(gold["pred_logits"]), "pred_boxes": torch.from_numpy(gold["pred_boxes"])}
        sizes = torch.tensor(POST_SIZES[:B])
        with torch.no_grad():
            res = post["bbox"](out, sizes)
        rec[name + "_sizes"] = sizes.numpy()
        rec[name + "_num_select"] = np.array([post["bbox"].num_select], dtype=np.int64)
        rec[name + "_scores"] = torch.stack([r["scores"] for r in res]).numpy()
        rec[name + "_labels"] = torch.stack([r["labels"] for r in res]).numpy()
        rec[name + "_boxes"] = torch.stack([r["boxes"] for r in res]).numpy()
        print("postprocess", name, rec[name + "_scores"].shape, "num_select", post["bbox"].num_select)
    np.savez_compressed(os.path.join(GOLD, "ref_postprocess.npz"), **rec)


PAD_VALID = [(640, 640), (576, 480)]              # (valid height, valid width) of the two images of the padded fixture


def padded_inputs():
    """Two images of different size padded to 640x640 the way util/misc.py:317-339 builds a NestedTensor."""
    x = synth_images(2, 9).clone()
    mask = torch.zeros(2, 640, 640, dtype=torch.bool)
    for b, (h, w) in enumerate(PAD_VALID):
        mask[b, h:, :] = True
        mask[b, :, w:] = True
        x[b][:, mask[b]] = 0
    return x, mask


def make_padded_golden():
    """Reference forward on a padded / mixed-size batch (masks not all False): pins the oracle's valid-ratio,
    proposal-masking and value-masking arithmetic (SURVEY.md 8f rank 3) ahead of the device implementation."""
    cfg = CONFIGS["tiny"]
    model, _, _ = ref_import.build_reference(cfg)
    model.load_state_dict(synth_state_dict(cfg, 5), strict=True)
    x, mask = padded_inputs()
    nested = sys.modules["_ref_util.misc"].NestedTensor(x, mask)
    with torch.no_grad():
        out = model(nested)
    np.savez_compressed(os.path.join(GOLD, "ref_tiny_padded.npz"), pred_logits=out["pred_logits"].numpy(),
                        pred_boxes=out["pred_boxes"].numpy(), enc_boxes=out["enc_outputs"]["pred_boxes"].numpy(),
                        valid=np.array(PAD_VALID, dtype=np.int64), meta=np.array([2, 5, 9], dtype=np.int64))
    print("padded", out["pred_logits"].shape)


def make_seed5_golden():
    """Reference forward of LW-DETR-tiny on a second set of weights / images (seeds 5 / 9, batch 2): the final predictions
    the oracle is compared with in tests/test_spec_and_oracle.py::test_oracle_matches_live_reference_with_forced_topk."""
    cfg = CONFIGS["tiny"]
    model, _, _ = ref_import.build_reference(cfg)
    model.load_state_dict(synth_state_dict(cfg, 5), strict=True)
    with torch.no_grad():
        out = model(synth_images(2, 9))
    np.savez_compressed(os.path.join(GOLD, "ref_tiny_seed5.npz"), pred_logits=out["pred_logits"].numpy(),
                        pred_boxes=out["pred_boxes"].numpy(), meta=np.array([2, 5, 9], dtype=np.int64))
    print("seed5", out["pred_logits"].shape)


# Inputs other than 640x640 (the reference's ViT resizes pos_embed to any token grid, vit.py:26-54, 343-358):
# (config, img_size, batch, height, width).  large at 1024x1024 takes the streaming top-k (S = 17408 > 16384) and the
# direct-gather deformable attention (P3 = 128x128 tokens); tiny at 512 runs natively with img_size = 512.
RES_CASES = [("tiny", 512, 2, 512, 512), ("small", 640, 1, 448, 768), ("large", 640, 1, 1024, 1024), ("xlarge", 640, 1, 768, 1344)]
RES_PADDED = ("tiny", 640, 832, 1344, [(800, 1333), (832, 1100)])   # COCO-style sizes (coco.py:111, max_size 1333), padded to 64
RES_IMAGE_SEED = 21


def res_golden_name(name, h, w, padded=False):
    return "ref_res_%s_%dx%d%s.npz" % (name, h, w, "_padded" if padded else "")


def res_padded_inputs():
    """Two differently sized images at the bottom / right of an 832x1344 canvas, with the NestedTensor mask."""
    name, _, H, W, sizes = RES_PADDED
    x = torch.zeros(len(sizes), 3, H, W)
    mask = torch.ones(len(sizes), H, W, dtype=torch.bool)
    for b, (h, w) in enumerate(sizes):
        x[b, :, :h, :w] = synth_images(1, RES_IMAGE_SEED + b, (h, w))[0]
        mask[b, :h, :w] = False
    return x, mask


def make_resolution_goldens():
    """Reference forward at input sizes other than 640x640, synthetic weights (seed WEIGHT_SEED) and images (seed
    RES_IMAGE_SEED): pins the oracle's grid, windows, position table and level shapes, and through it the device path."""
    for name, img_size, B, H, W in RES_CASES:
        cfg = dataclasses.replace(CONFIGS[name], img_size=img_size)
        model, _, _ = ref_import.build_reference(cfg)
        model.load_state_dict(synth_state_dict(cfg, WEIGHT_SEED), strict=True)
        with torch.no_grad():
            out = model(synth_images(B, RES_IMAGE_SEED, (H, W)))
        np.savez_compressed(os.path.join(GOLD, res_golden_name(name, H, W)), pred_logits=out["pred_logits"].numpy(),
                            pred_boxes=out["pred_boxes"].numpy(), enc_logits=out["enc_outputs"]["pred_logits"].numpy(),
                            enc_boxes=out["enc_outputs"]["pred_boxes"].numpy(),
                            meta=np.array([B, WEIGHT_SEED, RES_IMAGE_SEED, H, W, img_size], dtype=np.int64))
        print("resolution", name, H, W, out["pred_logits"].shape, flush=True)
    name, img_size, H, W, sizes = RES_PADDED
    cfg = dataclasses.replace(CONFIGS[name], img_size=img_size)
    model, _, _ = ref_import.build_reference(cfg)
    model.load_state_dict(synth_state_dict(cfg, WEIGHT_SEED), strict=True)
    x, mask = res_padded_inputs()
    with torch.no_grad():
        out = model(sys.modules["_ref_util.misc"].NestedTensor(x, mask))
    np.savez_compressed(os.path.join(GOLD, res_golden_name(name, H, W, padded=True)), pred_logits=out["pred_logits"].numpy(),
                        pred_boxes=out["pred_boxes"].numpy(), enc_boxes=out["enc_outputs"]["pred_boxes"].numpy(),
                        valid=np.array(sizes, dtype=np.int64),
                        meta=np.array([len(sizes), WEIGHT_SEED, RES_IMAGE_SEED, H, W, img_size], dtype=np.int64))
    print("resolution padded", name, H, W, out["pred_logits"].shape, flush=True)


def main():
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    if "--resolution-only" in sys.argv:
        make_resolution_goldens()
        return
    if "--seed5-only" in sys.argv:
        make_seed5_golden()
        return
    if "--postprocess-only" in sys.argv:
        make_postprocess_goldens()
        return
    if "--padded-only" in sys.argv:
        make_padded_golden()
        return
    for name, B in CASES:
        cfg = CONFIGS[name]
        model, _, _ = ref_import.build_reference(cfg)
        with open(os.path.join(GOLD, "state_dict_%s.json" % name), "w") as f:
            json.dump({k: list(v.shape) for k, v in model.state_dict().items()}, f, indent=0, sort_keys=True)
        model.load_state_dict(synth_state_dict(cfg, WEIGHT_SEED), strict=True)
        x = synth_images(B, IMAGE_SEED)
        rec = {}
        hooks = []
        enc = model.backbone[0].encoder
        for i, blk in enumerate(enc.blocks):
            hooks.append(blk.register_forward_hook(lambda m, a, o, i=i: rec.__setitem__("block%d" % i, sample(o))))

        def proj_hook(m, a, o):
            for l, f in enumerate(o):
                rec["level%d" % l] = sample(f.flatten(2).transpose(1, 2))

        hooks.append(model.backbone[0].projector.register_forward_hook(proj_hook))
        for i, lay in enumerate(model.transformer.decoder.layers):
            hooks.append(lay.register_forward_hook(lambda m, a, o, i=i: rec.__setitem__("dec%d" % i, sample(o))))
        hooks.append(model.transformer.decoder.ref_point_head.register_forward_hook(
            lambda m, a, o: rec.__setitem__("query_pos", sample(o))))
        with torch.no_grad():
            out = model(x)
        for h in hooks:
            h.remove()
        rec["pred_logits"] = out["pred_logits"].numpy()
        rec["pred_boxes"] = out["pred_boxes"].numpy()
        rec["enc_logits"] = out["enc_outputs"]["pred_logits"].numpy()
        rec["enc_boxes"] = out["enc_outputs"]["pred_boxes"].numpy()
        for i, a in enumerate(out["aux_outputs"]):
            rec["aux%d_logits" % i] = sample(a["pred_logits"], 8192)
            rec["aux%d_boxes" % i] = a["pred_boxes"].numpy()
        rec["meta"] = np.array([B, WEIGHT_SEED, IMAGE_SEED], dtype=np.int64)
        np.savez_compressed(os.path.join(GOLD, "ref_%s.npz" % name), **rec)
        print(name, "B=%d" % B, {k: v.shape for k, v in rec.items() if k.startswith("pred")})
    make_postprocess_goldens()
    make_padded_golden()
    make_seed5_golden()
    make_resolution_goldens()


if __name__ == "__main__":
    main()
