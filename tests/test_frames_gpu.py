"""GPU tests of the raw-frame input form: uint8 HWC frames of any size, resized on the device (antialiased bilinear) inside
the patch gather (csrc/resize.cu, lwdetr_resize_patches / lwdetr_forward_frames).  The specification every result is
compared with is tools/resize_spec.py."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import resize_spec  # noqa: E402
from test_model_gpu import TOL  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _engine(name, dt, wseed=1):
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS[name]
    eng = capi.Engine(cfg, dt)
    eng.load_state_dict(synth_state_dict(cfg, wseed))
    return cfg, eng


def _noise(h, w, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8))


def _crop_view(seed):
    """A 301 x 403 crop of a 500 x 700 surface whose rows are 2101 bytes apart and whose first byte sits at an odd address:
    neither the base pointer nor any row start is 16-byte aligned in general."""
    flat = torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (1 + 500 * 2101,), dtype=np.uint8)).cuda()
    view = flat.as_strided((301, 403, 3), (2101, 3, 1), 1 + 57 * 2101 + 31 * 3)
    assert view.data_ptr() % 16 != 0 and view.stride(0) % 2 == 1
    return view


def _mixed_frames(seed=0):
    """1080p, a small frame that is upscaled, a 4K frame, the odd-pitch crop and the smallest source the kernel takes."""
    return [_noise(1080, 1920, seed).cuda(), _noise(375, 500, seed + 1).cuda(), _noise(2160, 3840, seed + 2).cuda(), _crop_view(seed + 3),
            _noise(8, 8, seed + 4).cuda()]


def _ungather(A, B, H, W):
    """Window-major patch matrix [B*GH*GW, 768] (k = c*256 + py*16 + px) -> image [B, H, W, 3]."""
    from oracle import lwdetr_oracle as orc
    GH, GW = H // 16, W // 16
    x = orc.from_window_major(A.reshape(B * 16, -1, 768), B, GH, GW)                     # [B, GH, GW, 768]
    return x.reshape(B, GH, GW, 3, 16, 16).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, 3)


def _check_against_spec(got, frames, dsts, size, dt):
    """got [B, H, W, 3] (float, the kernel's values) against the spec: equal, except that a pixel whose pre-rounding value lies
    within 1e-3 of a half level may land on the neighbouring level; such pixels are fewer than 1e-4 of all.  Returns the
    number of differing pixels."""
    H, W = size
    total = bad = 0
    for b, (fr, (dh, dw)) in enumerate(zip(frames, dsts)):
        lv = resize_spec.resize_levels(fr.cpu().numpy(), dh, dw)
        u8 = resize_spec.round_levels(lv).astype(np.int32)
        cast = lambda lev: torch.from_numpy(resize_spec.normalise(np.clip(lev, 0, 255), MEAN, STD)).to(dt).float()
        g = got[b, :dh, :dw]
        diff = g != cast(u8)
        if diff.any():
            tie = torch.from_numpy(resize_spec.tie_pixels(lv))
            assert not (diff & ~tie).any(), "frame %d differs from the spec away from a rounding tie" % b
            neighbour = (g == cast(u8 + 1)) | (g == cast(u8 - 1))
            assert neighbour[diff].all(), "frame %d: a tie pixel is more than one level off" % b
        assert (got[b, dh:] == 0).all() and (got[b, :, dw:] == 0).all(), "frame %d: padding is not exactly 0" % b
        total += diff.numel()
        bad += int(diff.sum())
    assert bad < 1e-4 * total, (bad, total)
    return bad


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_kernel_matches_the_spec_on_mixed_frames(dt):
    from b200 import capi
    frames = _mixed_frames()
    size = (640, 640)
    dsts = [(640, 640), (640, 640), (640, 640), (640, 640), (640, 640)]
    A, _ = capi.resize_patches(frames, dsts, size, dt)
    torch.cuda.synchronize()
    _check_against_spec(_ungather(A.float().cpu(), len(frames), *size), frames, dsts, size, dt)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_kernel_pads_and_builds_the_mask(dt):
    """Frames with their own dst sizes on a non-square canvas (one tile row and tile column only partly covered, one frame
    16x downscaled): values, zero padding and the device-made mask."""
    from b200 import capi
    frames = [_noise(1080, 1920, 7).cuda(), _crop_view(8), _noise(2048, 3000, 9).cuda(), _noise(50, 40, 10).cuda()]
    size = (448, 768)
    dsts = [(432, 768), (301, 403), (128, 200), (448, 7)]
    A, mask = capi.resize_patches(frames, dsts, size, dt, want_mask=True)
    torch.cuda.synchronize()
    _check_against_spec(_ungather(A.float().cpu(), len(frames), *size), frames, dsts, size, dt)
    want = torch.ones(len(frames), *size, dtype=torch.bool)
    for b, (dh, dw) in enumerate(dsts):
        want[b, :dh, :dw] = False
    assert torch.equal(mask.cpu(), want)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("size", [(640, 640), (448, 768)])
def test_identity_size_is_bit_identical_to_the_uint8_path(size, dt):
    """Frames already at the run size: the patch matrix and the predictions equal those of Engine.forward(uint8)."""
    cfg, eng = _engine("tiny", dt)
    B, (H, W) = 2, size
    u8 = torch.stack([_noise(H, W, 20 + b) for b in range(B)]).cuda()
    n = B * (H // 16) * (W // 16) * 768
    eng.capture("patch_gather", n)
    a = {k: v.clone() for k, v in eng.forward(u8, want_aux=False).items()}
    pa = eng.capture_results()["patch_gather"].clone()
    b = eng.forward_frames(u8, size=size, want_aux=False)
    torch.cuda.synchronize()
    pb = eng.capture_results()["patch_gather"]
    eng.clear_captures()
    assert torch.equal(pa, pb)
    assert torch.equal(a["pred_logits"], b["pred_logits"]) and torch.equal(a["pred_boxes"], b["pred_boxes"])
    eng.close()


def _compare_predictions(free, forced, want, cfg, dt):
    """Runs whose inputs differ in at most a few tie pixels.  Free-running, the two-stage selection is the same set (>= 99 %;
    near-equal scores may swap slots, and a slot carries its own learned query).  With the selection forced to `want`'s,
    the predictions agree within the fp16 / bf16 bars of test_model_gpu."""
    tol = TOL[dt]
    ta, tb = free["topk_index"].cpu(), want["topk_index"].cpu()
    for i in range(ta.shape[0]):
        assert len(set(ta[i].tolist()) & set(tb[i].tolist())) >= 0.99 * cfg.num_queries
    assert torch.equal(forced["topk_index"], want["topk_index"])
    assert torch.isfinite(forced["pred_logits"]).all() and torch.isfinite(forced["pred_boxes"]).all()
    assert (forced["pred_logits"] - want["pred_logits"]).abs().max().item() <= tol["logits_abs"]
    assert (forced["pred_boxes"] - want["pred_boxes"]).abs().max().item() <= tol["boxes"]


@pytest.mark.parametrize("name", ["tiny", "large"])
def test_forward_frames_matches_forward_on_spec_resized_frames(name):
    dt = torch.float16
    cfg, eng = _engine(name, dt)
    frames = _mixed_frames(30)
    u8 = torch.stack([torch.from_numpy(resize_spec.resize_u8(f.cpu().numpy(), 640, 640)) for f in frames]).cuda()
    want = eng.forward(u8)
    free = eng.forward_frames(frames)
    forced = eng.forward_frames(frames, topk_override=want["topk_index"])
    torch.cuda.synchronize()
    _compare_predictions(free, forced, want, cfg, dt)
    eng.close()


def test_keep_aspect_batch_is_padded_and_masked_on_the_device():
    """480x640 and 1080x1920 at short side 800 / max side 1333 -> 800x1066 and 750x1333 on an 832x1344 canvas: the patch
    matrix follows the spec with exact zeros outside the frames, and the predictions are those of the existing path fed
    the spec's zero-padded normalised canvas and its mask."""
    dt = torch.float16
    cfg, eng = _engine("tiny", dt)
    frames = [_noise(480, 640, 40).cuda(), _noise(1080, 1920, 41).cuda()]
    H, W, B = 832, 1344, 2
    eng.capture("patch_gather", B * (H // 16) * (W // 16) * 768)
    got = eng.forward_frames(frames, fit="keep_aspect", short_side=800, max_side=1333)
    torch.cuda.synchronize()
    dsts = got["frame_sizes"]
    assert dsts == [(800, 1066), (750, 1333)]
    got = {k: v.clone() for k, v in got.items() if isinstance(v, torch.Tensor)}
    pg = eng.capture_results()["patch_gather"].clone()
    eng.clear_captures()
    differing = _check_against_spec(_ungather(pg, B, H, W), frames, dsts, (H, W), dt)
    canvas, _, mask = resize_spec.canvas([f.cpu().numpy() for f in frames], dsts, (H, W), MEAN, STD)
    x = torch.from_numpy(canvas).permute(0, 3, 1, 2).contiguous().cuda()
    want = eng.forward(x, mask=torch.from_numpy(mask).cuda())
    torch.cuda.synchronize()
    if differing == 0:
        assert torch.equal(got["pred_logits"], want["pred_logits"]) and torch.equal(got["pred_boxes"], want["pred_boxes"])
    forced = eng.forward_frames(frames, fit="keep_aspect", short_side=800, max_side=1333, topk_override=want["topk_index"])
    torch.cuda.synchronize()
    _compare_predictions(got, forced, want, cfg, dt)
    # the mask matters: without it the same canvas gives other predictions
    plain = eng.forward(x)
    assert not torch.equal(plain["pred_boxes"], want["pred_boxes"])
    eng.close()


def test_source_sizes_neither_replan_nor_recapture():
    """With CUDA graphs on, batches of different source sizes (and an unpadded -> padded -> unpadded sequence) at one run
    size reuse the plan: the op table is unchanged, and every result equals that of a fresh engine."""
    dt = torch.float16
    batches = [dict(frames=[_noise(480, 640, 50).cuda(), _noise(1080, 1920, 51).cuda()]),
               dict(frames=[_noise(720, 1280, 52).cuda(), _crop_view(53)]),
               dict(frames=[_noise(600, 400, 54).cuda(), _noise(375, 500, 55).cuda()], fit="keep_aspect", short_side=640, max_side=640),
               dict(frames=[_noise(2160, 3840, 56).cuda(), _noise(64, 64, 57).cuda()])]
    fresh = []
    for kw in batches:
        _, e = _engine("small", dt)
        o = e.forward_frames(want_aux=False, **kw)
        fresh.append({k: o[k].clone() for k in ("pred_logits", "pred_boxes")})
        e.close()
    _, eng = _engine("small", dt)
    eng.set_option("cuda_graph", 1)
    ops0 = None
    for rep in range(3):                                   # eager first run of the plan, then graph capture, then replay
        for kw, want in zip(batches, fresh):
            o = eng.forward_frames(want_aux=False, **kw)
            torch.cuda.synchronize()
            assert torch.equal(o["pred_logits"], want["pred_logits"]) and torch.equal(o["pred_boxes"], want["pred_boxes"]), rep
            ops = eng.ops()
            ops0 = ops if ops0 is None else ops0
            assert ops == ops0 and "patch_gather" in [lab for lab, _, _ in ops]
    eng.close()


def test_detect_returns_boxes_in_each_frames_own_pixels():
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR, PostProcess
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    model.cuda()
    frames = [_noise(480, 640, 60).cuda(), _noise(1080, 1920, 61).cuda(), _noise(300, 200, 62).cuda()]
    for kw in (dict(), dict(fit="keep_aspect", short_side=512, max_side=704)):
        out = model.forward_frames(frames, **kw)
        assert out["pred_logits"].shape == (3, cfg.num_queries, cfg.num_classes) and "aux_outputs" in out
        det = model.detect(frames, num_select=50, **kw)
        sizes = torch.tensor([[480.0, 640.0], [1080.0, 1920.0], [300.0, 200.0]], device="cuda")
        want = PostProcess(50)(out, sizes)
        for d, w, (h, wd) in zip(det, want, sizes.tolist()):
            assert d["boxes"].shape == (50, 4)
            assert torch.equal(d["scores"], w["scores"]) and torch.equal(d["labels"], w["labels"]) and torch.equal(d["boxes"], w["boxes"])
        # boxes scale with the frame: the same predictions at unit size, times (w, h, w, h)
        unit = PostProcess(50)(out, torch.ones(3, 2, device="cuda"))
        for d, u, (h, wd) in zip(det, unit, sizes.tolist()):
            assert torch.allclose(d["boxes"], u["boxes"] * torch.tensor([wd, h, wd, h], device="cuda"), rtol=1e-6, atol=1e-3)
    assert len(model.detect(torch.stack([frames[0], frames[0]]))) == 2        # one [B, h, w, 3] tensor works too


def test_rejections_name_the_limit():
    from b200 import capi
    dt = torch.float16
    z = lambda h, w: torch.zeros(h, w, 3, dtype=torch.uint8, device="cuda")
    for frames, dsts, msg in (([z(2064, 64)], [(128, 64)], "factor above 16"), ([z(64, 2064)], [(64, 128)], "factor above 16"),
                              ([z(4, 64)], [(64, 64)], r"\[8, 8192\]"), ([z(64, 64)], [(192, 64)], "run size 128x128"),
                              ([z(64, 64)], [(64, 0)], "run size 128x128")):
        with pytest.raises(RuntimeError, match=msg):
            capi.resize_patches(frames, dsts, (128, 128), dt)
    cfg, eng = _engine("tiny", dt)
    for frames, kw, msg in ((z(64, 128)[:, ::2], {}, "stride"), (z(64, 64).permute(1, 0, 2)[:, :32], {}, "stride"),
                            (torch.zeros(64, 64, 3, device="cuda"), {}, "uint8"), (z(64, 64).cpu(), {}, "CUDA"),
                            (z(64, 64), dict(size=(640, 600)), "multiples of 64"), (z(64, 64), dict(size=(1408, 640)), "1344"),
                            (z(12000, 64)[:11000], {}, r"\[8, 8192\]"), (z(64, 64), dict(fit="keep_aspect", short_side=2), "factor above 16")):
        with pytest.raises(RuntimeError, match=msg):
            eng.forward_frames([frames], **kw)
    o = eng.forward_frames([z(64, 64)], want_aux=False)             # the engine still runs after the rejected calls
    torch.cuda.synchronize()
    assert torch.isfinite(o["pred_logits"]).all()
    eng.close()
