"""CPU tests of the raw-frame input form (forward_frames): the resize filter's restatement (tools/resize_spec.py) against
torch's antialiased interpolate and PIL, the keep-aspect size rule against hand-worked cases of the reference's, and the
host-side checks that need no GPU."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import resize_spec  # noqa: E402
from b200 import capi  # noqa: E402
from b200.config import CONFIGS, frame_sizes, keep_aspect_size  # noqa: E402

# (source, destination): upscale, identity, non-integer and integer downscale, > 8x downscale, non-square both ways
SIZES = [((375, 500), (640, 640)), ((64, 96), (64, 96)), ((1080, 1920), (640, 640)), ((480, 640), (640, 640)),
         ((720, 1280), (448, 768)), ((1100, 1500), (128, 128)), ((8, 8), (128, 192)), ((300, 200), (100, 333)),
         ((2160, 3840), (640, 640))]


def _noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("src,dst", SIZES)
def test_spec_matches_torch_antialias_interpolate(src, dst):
    img = _noise(src[0], src[1], 1)
    got = resize_spec.resize_levels(img, dst[0], dst[1])
    x = torch.from_numpy(img).permute(2, 0, 1)[None].float()
    want = F.interpolate(x, size=dst, mode="bilinear", align_corners=False, antialias=True)[0].permute(1, 2, 0).numpy()
    assert np.abs(got - want).max() <= 1e-3


@pytest.mark.parametrize("src,dst", SIZES[:8])
def test_rounded_spec_is_within_one_level_of_pil(src, dst):
    Image = pytest.importorskip("PIL.Image")
    img = _noise(src[0], src[1], 2)
    got = resize_spec.resize_u8(img, dst[0], dst[1]).astype(np.int32)
    want = np.asarray(Image.fromarray(img).resize((dst[1], dst[0]), Image.BILINEAR)).astype(np.int32)
    assert np.abs(got - want).max() <= 1


def test_identity_size_returns_the_input():
    img = _noise(72, 136, 3)
    assert np.array_equal(resize_spec.resize_u8(img, 72, 136), img)
    w = resize_spec.axis_weights(136, 136)
    assert np.array_equal(w, np.eye(136, dtype=np.float32))          # every tap weight is exactly 1 or 0


def test_tap_count_bound():
    """At the largest downscale factor the kernel accepts (16) an output has at most 33 taps."""
    for n_in, n_out in ((8192, 512), (1024, 64), (2047, 128)):
        assert (resize_spec.axis_weights(n_in, n_out) > 0).sum(1).max() <= 33


def test_canvas_pads_with_zero_after_normalisation():
    fr = [_noise(40, 60, 4), _noise(90, 50, 5)]
    out, u8, mask = resize_spec.canvas(fr, [(64, 96), (128, 70)], (128, 128), capi.IMAGENET_MEAN, capi.IMAGENET_STD)
    assert (out[0, 64:] == 0).all() and (out[0, :, 96:] == 0).all() and (out[1, :, 70:] == 0).all()
    assert mask[0, :64, :96].sum() == 0 and mask[0].sum() == 128 * 128 - 64 * 96 and mask[1].sum() == 128 * (128 - 70)
    assert np.array_equal(u8[1, :128, :70], resize_spec.resize_u8(fr[1], 128, 70))


@pytest.mark.parametrize("hw,want", [((480, 640), (800, 1066)), ((640, 480), (1066, 800)), ((500, 1500), (444, 1332)),
                                     ((800, 1200), (800, 1200)), ((1080, 1920), (750, 1333)), ((1200, 800), (1200, 800))])
def test_keep_aspect_size_hand_worked(hw, want):
    """datasets/transforms.py:97-115 at size 800, max_size 1333: 480x640 -> the shorter side to 800, int(800 * 640 / 480) =
    1066; 500x1500 hits the cap: size = round(1333 * 500 / 1500) = 444, int(444 * 1500 / 500) = 1332; a shorter side that is
    already 800 returns the image's size."""
    assert keep_aspect_size(hw[0], hw[1], 800, 1333) == want


def test_frame_sizes():
    cfg = CONFIGS["tiny"]
    assert frame_sizes(cfg, [(1080, 1920), (375, 500)]) == ((640, 640), [(640, 640)] * 2)
    assert frame_sizes(cfg, [(1080, 1920)], size=(448, 768)) == ((448, 768), [(448, 768)])
    assert frame_sizes(cfg, [(480, 640), (1080, 1920)], fit="keep_aspect", short_side=800, max_side=1333) == \
        ((832, 1344), [(800, 1066), (750, 1333)])
    assert frame_sizes(cfg, [(480, 640)], fit="keep_aspect", short_side=320) == ((640, 640), [(320, 426)])
    with pytest.raises(RuntimeError, match="multiples of 64"):
        frame_sizes(cfg, [(480, 640)], size=(600, 640))
    with pytest.raises(RuntimeError, match="does not fit"):
        frame_sizes(cfg, [(480, 640)], size=(640, 640), fit="keep_aspect", short_side=800, max_side=1333)
    with pytest.raises(RuntimeError, match="1344"):
        frame_sizes(cfg, [(480, 640)], fit="keep_aspect", short_side=1400)
    with pytest.raises(RuntimeError, match="short_side"):
        frame_sizes(cfg, [(480, 640)], fit="keep_aspect")
    with pytest.raises(RuntimeError, match="fit must be"):
        frame_sizes(cfg, [(480, 640)], fit="crop")


def test_frame_list_rejects_what_the_kernel_cannot_read():
    with pytest.raises(RuntimeError, match="uint8"):
        capi.frame_list([torch.zeros(16, 16, 3)])
    with pytest.raises(RuntimeError, match="HWC"):
        capi.frame_list([torch.zeros(3, 16, 16, dtype=torch.uint8)])
    with pytest.raises(RuntimeError, match="CUDA"):
        capi.frame_list([torch.zeros(16, 16, 3, dtype=torch.uint8)])
    with pytest.raises(RuntimeError, match="no frames"):
        capi.frame_list([])


def test_frame_struct_matches_the_header():
    """lwdetr_frame in include/lwdetr_b200.h: pointer, two int32, int64 pitch, two int32 = 32 bytes, natural alignment."""
    import ctypes
    assert ctypes.sizeof(capi.FrameStruct) == 32
    assert [capi.FrameStruct.pitch_bytes.offset, capi.FrameStruct.dst_h.offset, capi.FrameStruct.dst_w.offset] == [16, 24, 28]
    with open(os.path.join(ROOT, "include", "lwdetr_b200.h")) as f:
        hdr = f.read()
    assert "lwdetr_forward_frames" in hdr and "lwdetr_resize_patches" in hdr
    assert {"lwdetr_forward_frames", "lwdetr_resize_patches"} <= set(capi.exported_symbols())


def test_kernel_level_entry_rejects_bad_frames_without_a_gpu():
    """The C ABI's own checks run before anything is launched, so they can be exercised on a machine without a GPU."""
    import ctypes
    fr = (capi.FrameStruct * 1)()
    norm = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    dummy = ctypes.c_void_p(256)                                  # never dereferenced: every call below is rejected

    def call(h, w, pitch, dh, dw, H=128, W=128):
        fr[0].data, fr[0].height, fr[0].width, fr[0].pitch_bytes, fr[0].dst_h, fr[0].dst_w = 256, h, w, pitch, dh, dw
        rc = capi.lib().lwdetr_resize_patches(capi.F16, ctypes.cast(fr, ctypes.c_void_p), 1, H, W, ctypes.cast(norm, ctypes.c_void_p),
                                              ctypes.cast(norm, ctypes.c_void_p), dummy, None, None)
        return rc, capi.lib().lwdetr_last_error().decode()

    for args, msg in (((2064, 64, 192, 128, 64), "factor above 16"), ((4, 64, 192, 64, 64), "[8, 8192]"),
                      ((64, 9000, 27000, 64, 128), "[8, 8192]"), ((64, 64, 100, 64, 64), "pitch_bytes"),
                      ((64, 64, 192, 192, 64), "run size 128x128"), ((64, 64, 192, 0, 64), "run size 128x128")):
        rc, err = call(*args)
        assert rc != 0 and msg in err, (args, err)
    rc, err = call(64, 64, 192, 64, 64, H=100)
    assert rc != 0 and "multiples of 64" in err
