"""GPU tests of the NV12 frame input (lwdetr_resize_patches_nv12 / lwdetr_forward_frames_nv12): every result must be
bit-identical to the RGB frame path fed tools/yuv_spec.py's conversion of the same frames."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import yuv_spec  # noqa: E402

CS4 = ["bt601", "bt709", "bt601_full", "bt709_full"]


def _engine(name, dt, wseed=1):
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    cfg = CONFIGS[name]
    eng = capi.Engine(cfg, dt)
    eng.load_state_dict(synth_state_dict(cfg, wseed))
    return cfg, eng


def _nv12(h, w, seed):
    """(luma [h, w], chroma [ceil(h/2), 2 * ceil(w/2)]) random CUDA planes."""
    rng = np.random.default_rng(seed)
    luma = rng.integers(0, 256, (h, w), dtype=np.uint8)
    chroma = rng.integers(0, 256, ((h + 1) // 2, 2 * ((w + 1) // 2)), dtype=np.uint8)
    return torch.from_numpy(luma).cuda(), torch.from_numpy(chroma).cuda()


def _crop_pair(seed):
    """A 301 x 403 crop of a larger NV12 surface: luma and chroma are separate allocations, both with odd pitches (701 and
    809 bytes) and bases at odd addresses."""
    rng = np.random.default_rng(seed)
    lflat = torch.from_numpy(rng.integers(0, 256, (1 + 500 * 701,), dtype=np.uint8)).cuda()
    cflat = torch.from_numpy(rng.integers(0, 256, (3 + 260 * 809,), dtype=np.uint8)).cuda()
    luma = lflat.as_strided((301, 403), (701, 1), 1 + 57 * 701 + 31)
    chroma = cflat.as_strided((151, 404), (809, 1), 3 + 20 * 809 + 18)
    assert luma.data_ptr() % 2 == 1 and chroma.data_ptr() % 2 == 1
    return luma, chroma


def _rgb(pair, cs):
    """The spec's RGB frame of an NV12 frame, as a CUDA uint8 [h, w, 3] tensor."""
    return torch.from_numpy(yuv_spec.nv12_to_rgb(pair[0].cpu().numpy(), pair[1].cpu().numpy(), cs)).cuda()


def _packed(pair):
    return torch.cat([pair[0], pair[1]])


def _mixed():
    """1080p, an odd-width upscale, 4K, the smallest source, 16x downscale, and the unaligned crop."""
    return [_nv12(1080, 1920, 0), _nv12(375, 501, 1), _nv12(2160, 3840, 2), _nv12(8, 8, 3), _nv12(2048, 3000, 4), _crop_pair(5)]


def _check_kernel(frames, dsts, size, dt, cs):
    from b200 import capi
    cs_list = [cs] * len(frames) if isinstance(cs, str) else cs
    A, mask = capi.resize_patches(frames, dsts, size, dt, want_mask=True, colorspace=cs)
    B_, mask_b = capi.resize_patches([_rgb(f, c) for f, c in zip(frames, cs_list)], dsts, size, dt, want_mask=True)
    torch.cuda.synchronize()
    assert torch.equal(A, B_)
    assert torch.equal(mask, mask_b)
    return A


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_kernel_equals_the_rgb_path_on_converted_frames(dt):
    dsts = [(640, 640)] * 4 + [(128, 188), (640, 640)]                 # 2048 x 3000 -> 128 x 188: 16x per axis
    A = _check_kernel(_mixed(), dsts, (640, 640), dt, "bt709")
    assert torch.isfinite(A.float()).all()


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_kernel_every_colorspace_with_padding(dt):
    frames = [_nv12(1080, 1920, 10), _crop_pair(11), _nv12(2048, 3000, 12), _nv12(51, 41, 13)]
    _check_kernel(frames, [(432, 768), (301, 403), (128, 200), (448, 7)], (448, 768), dt, CS4)


def test_kernel_two_launch_groups():
    """70 small frames of odd and even sizes, mixed colorspaces, some padded: more than one group of 64 descriptors."""
    rng = np.random.default_rng(30)
    frames = [_nv12(int(rng.integers(8, 90)), int(rng.integers(8, 90)), 100 + i) for i in range(70)]
    dsts = [(128, 128) if i % 3 else (int(rng.integers(8, 129)), int(rng.integers(8, 129))) for i in range(70)]
    _check_kernel(frames, dsts, (128, 128), torch.float16, [CS4[i % 4] for i in range(70)])


def _flat(out):
    t = [out["pred_logits"], out["pred_boxes"], out["topk_index"], out["enc_outputs"]["pred_logits"], out["enc_outputs"]["pred_boxes"]]
    for a in out["aux_outputs"]:
        t += [a["pred_logits"], a["pred_boxes"]]
    return [x.clone() for x in t]


def _equal(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_forward_frames_equals_rgb_and_alternates_under_graphs():
    """tiny, CUDA graphs on: NV12 and RGB-of-spec batches alternate at one (B, H, W) through eager, capture and replay; every
    output is bit-identical and the op table never changes."""
    _, eng = _engine("tiny", torch.float16)
    eng.set_option("cuda_graph", 1)
    frames = [_nv12(1080, 1920, 20), _nv12(375, 501, 21), _crop_pair(22), _nv12(720, 1280, 23)]
    cs = ["bt709", "bt601", "bt709_full", "bt601_full"]
    rgb = [_rgb(f, c) for f, c in zip(frames, cs)]
    ops0 = want = None
    for rep in range(3):
        a = _flat(eng.forward_frames(rgb))
        b = _flat(eng.forward_frames(frames, colorspace=cs))
        torch.cuda.synchronize()
        want = a if want is None else want
        assert _equal(a, want) and _equal(b, want), rep
        ops0 = eng.ops() if ops0 is None else ops0
        assert eng.ops() == ops0
    eng.close()


def test_packed_form_equals_pair_form():
    _, eng = _engine("tiny", torch.float16)
    pairs = [_nv12(480, 640, 40), _nv12(480, 640, 41)]
    want = _flat(eng.forward_frames(pairs, colorspace="bt601"))
    got_list = _flat(eng.forward_frames([_packed(p) for p in pairs], colorspace="bt601"))
    got_batch = _flat(eng.forward_frames(torch.stack([_packed(p) for p in pairs]), colorspace="bt601"))
    torch.cuda.synchronize()
    assert _equal(got_list, want) and _equal(got_batch, want)
    eng.close()


def test_keep_aspect_equals_rgb():
    _, eng = _engine("tiny", torch.float16)
    frames = [_nv12(480, 640, 50), _crop_pair(51), _nv12(1080, 1920, 52)]
    cs = ["bt709", "bt709_full", "bt601"]
    kw = dict(fit="keep_aspect", short_side=512, max_side=704)
    a = eng.forward_frames([_rgb(f, c) for f, c in zip(frames, cs)], **kw)
    sa = a["frame_sizes"]
    a = _flat(a)
    b = eng.forward_frames(frames, colorspace=cs, **kw)
    torch.cuda.synchronize()
    assert b["frame_sizes"] == sa and len(set(sa)) > 1                           # frames of different sizes: the batch is padded
    assert _equal(_flat(b), a)
    eng.close()


def test_detect_on_nv12_equals_rgb():
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    model.cuda()
    frames = [_nv12(480, 640, 60), _nv12(1080, 1920, 61), _crop_pair(62)]
    rgb = [_rgb(f, "bt709") for f in frames]
    for kw in (dict(), dict(fit="keep_aspect", short_side=512, max_side=704)):
        want = model.detect(rgb, num_select=50, **kw)
        got = model.detect(frames, num_select=50, colorspace="bt709", **kw)
        for g, w in zip(got, want):
            assert torch.equal(g["scores"], w["scores"]) and torch.equal(g["labels"], w["labels"]) and torch.equal(g["boxes"], w["boxes"])


def test_rejections_on_the_device():
    from b200 import capi
    _, eng = _engine("tiny", torch.float16)
    luma, chroma = _nv12(51, 41, 70)
    for frames, kw, msg in (([(luma, chroma[:, :40])], dict(colorspace="bt601"), r"chroma must be \[26, 42\]"),
                            ([(luma, chroma[:25])], dict(colorspace="bt601"), r"chroma must be \[26, 42\]"),
                            ([(luma[:, ::2], chroma)], dict(colorspace="bt601"), "luma has strides"),
                            ([_packed(_nv12(64, 64, 71))[:, :63]], dict(colorspace="bt601"), "h and w even"),
                            ([(luma, chroma)], {}, "need colorspace"),
                            ([(luma, chroma), _rgb((luma, chroma), 0)], dict(colorspace="bt601"), "not a mix"),
                            ([_rgb((luma, chroma), 0)], dict(colorspace="bt601"), "NV12 frames only"),
                            ([(luma, chroma)], dict(colorspace="bt601", fit="keep_aspect", short_side=2), "factor above 16")):
        with pytest.raises(RuntimeError, match=msg):
            eng.forward_frames(frames, **kw)
    o = eng.forward_frames([(luma, chroma)], want_aux=False, colorspace="bt601")    # the engine still runs after the rejected calls
    torch.cuda.synchronize()
    assert torch.isfinite(o["pred_logits"]).all()
    eng.close()
