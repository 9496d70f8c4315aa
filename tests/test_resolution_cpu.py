"""CPU tests of inference at input sizes other than 640x640: the oracle against golden outputs of the UNMODIFIED reference
at those sizes (tools/make_goldens.py --resolution-only), the non-square host bicubic resize, and the grid rule that
decides the size a batch runs at."""
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))

from b200 import capi  # noqa: E402
from b200.config import CONFIGS, check_input_size, run_size  # noqa: E402
from b200.synth import synth_images, synth_state_dict  # noqa: E402
from oracle import lwdetr_oracle as orc  # noqa: E402

import oracle_hw  # noqa: E402

RES_CASES = [("tiny", 512, 512), ("small", 448, 768), ("large", 1024, 1024), ("xlarge", 768, 1344)]


def _close(a, b, atol, what):
    err = np.abs(np.asarray(a) - np.asarray(b)).max()
    assert err <= atol, "%s: %g" % (what, err)


@pytest.mark.parametrize("name,H,W", RES_CASES)
def test_oracle_matches_reference_at_resolution(name, H, W):
    g = np.load(os.path.join(GOLD, "ref_res_%s_%dx%d.npz" % (name, H, W)))
    B, wseed, iseed, gh, gw, img_size = (int(v) for v in g["meta"])
    assert (gh, gw) == (H, W)
    cfg = dataclasses.replace(CONFIGS[name], img_size=img_size)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = oracle_hw.forward(synth_state_dict(cfg, wseed), cfg, synth_images(B, iseed, (H, W)))
    assert out["pred_logits"].shape == g["pred_logits"].shape
    _close(out["pred_logits"], g["pred_logits"], 1e-4, "pred_logits")
    _close(out["pred_boxes"], g["pred_boxes"], 1e-4, "pred_boxes")
    _close(out["enc_outputs"]["pred_logits"], g["enc_logits"], 1e-4, "enc logits")
    _close(out["enc_outputs"]["pred_boxes"], g["enc_boxes"], 1e-4, "enc boxes")


def test_oracle_matches_reference_on_padded_coco_sized_batch():
    """800x1333 and 832x1100 images on an 832x1344 canvas with the NestedTensor mask."""
    import make_goldens
    g = np.load(os.path.join(GOLD, "ref_res_tiny_832x1344_padded.npz"))
    B, wseed, iseed, H, W, img_size = (int(v) for v in g["meta"])
    assert [tuple(v) for v in g["valid"].tolist()] == make_goldens.RES_PADDED[4] and (H, W) == (832, 1344)
    cfg = dataclasses.replace(CONFIGS["tiny"], img_size=img_size)
    x, mask = make_goldens.res_padded_inputs()
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = oracle_hw.forward(synth_state_dict(cfg, wseed), cfg, x, mask=mask)
    _close(out["pred_logits"], g["pred_logits"], 1e-4, "pred_logits")
    _close(out["pred_boxes"], g["pred_boxes"], 1e-4, "pred_boxes")
    _close(out["enc_outputs"]["pred_boxes"], g["enc_boxes"], 1e-4, "enc boxes")


def test_size_aware_oracle_at_the_configured_size_is_the_oracle():
    """At 640x640 the size-aware ViT and level shapes reproduce the oracle's bit for bit, and forward() is the oracle's."""
    cfg = CONFIGS["tiny"]
    sd = synth_state_dict(cfg, 1)
    x = synth_images(1, 0)
    a, b = {}, {}
    ta = oracle_hw.vit_encoder_hw(x, sd, cfg, a)
    tb = orc.vit_encoder(x, sd, cfg, b)
    assert all(torch.equal(p, q) for p, q in zip(ta, tb)) and torch.equal(a["patch"], b["patch"])
    for name in CONFIGS:
        assert oracle_hw.AtInputSize(CONFIGS[name], 640, 640).level_shapes == CONFIGS[name].level_shapes
    g = np.load(os.path.join(GOLD, "ref_tiny.npz"))
    B, wseed, iseed = (int(v) for v in g["meta"])
    out = oracle_hw.forward(synth_state_dict(cfg, wseed), cfg, synth_images(B, iseed))
    _close(out["pred_logits"], g["pred_logits"], 1e-4, "pred_logits")
    _close(out["pred_boxes"], g["pred_boxes"], 1e-5, "pred_boxes")


@pytest.mark.parametrize("out_h,out_w", [(40, 84), (28, 48), (84, 16), (14, 14), (9, 5)])
def test_host_bicubic_hw_matches_torch(out_h, out_w):
    g = torch.Generator().manual_seed(out_h * 100 + out_w)
    src = torch.randn(14, 14, 7, generator=g)
    ref = F.interpolate(src.permute(2, 0, 1)[None], size=(out_h, out_w), mode="bicubic", align_corners=False)[0].permute(1, 2, 0)
    got = capi.host_bicubic_hw(src, out_h, out_w)
    assert got.shape == (out_h, out_w, 7)
    assert (got - ref).abs().max().item() < 2e-5
    if out_h == out_w:                                         # the square entry point is the same function
        assert torch.equal(got, capi.host_bicubic(src, out_h))


def test_grid_rule():
    tiny, large = CONFIGS["tiny"], CONFIGS["large"]
    assert run_size(tiny, 640, 640) == (640, 640)
    assert run_size(tiny, 480, 600) == (640, 640)                 # smaller batches keep the configured size
    assert run_size(tiny, 800, 1333) == (832, 1344)               # COCO eval size: each side up to a multiple of 64
    assert run_size(tiny, 700, 900) == (704, 960)                 # not a multiple of 64: rounded up, padded
    assert run_size(large, 1024, 1024) == (1024, 1024)
    assert run_size(dataclasses.replace(tiny, img_size=512), 512, 896) == (512, 896)
    for h, w in ((1345, 640), (640, 1400), (2000, 2000)):        # oversize
        with pytest.raises(RuntimeError, match="1344"):
            run_size(tiny, h, w)
    assert large.level_shapes_at(1024, 1024) == ((128, 128), (32, 32))
    assert large.level_shapes_at(768, 1344) == ((96, 168), (24, 42))
    assert tiny.level_shapes_at(448, 768) == ((28, 48),)
    assert large.level_shapes_at(640, 640) == large.level_shapes and large.memory_len_at(640, 640) == large.memory_len


def test_input_size_checks():
    small = CONFIGS["small"]
    check_input_size(small, 256, 1344)
    for h, w in ((640, 650), (100, 640), (64, 640), (1408, 640)):
        with pytest.raises(RuntimeError, match="multiples of 64"):
            check_input_size(small, h, w)
    with pytest.raises(RuntimeError, match="num_queries"):
        check_input_size(small, 128, 256)                         # 8x16 = 128 memory tokens < 300 queries
