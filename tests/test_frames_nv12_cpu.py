"""CPU tests of the NV12 frame input: the conversion's restatement (tools/yuv_spec.py) against OpenCV and float64, the C ABI's
host checks of lwdetr_frame_nv12, and the Python side's rejections, none of which needs a GPU."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import yuv_spec  # noqa: E402
from b200 import capi  # noqa: E402


def _all_triples():
    """Every (Y, U, V) once: Y, U, V uint8 arrays of 2^24 elements."""
    n = np.arange(1 << 24, dtype=np.uint32)
    return (n & 255).astype(np.uint8), (n >> 16).astype(np.uint8), ((n >> 8) & 255).astype(np.uint8)


def test_bt601_limited_is_opencv_over_every_triple():
    """A 4096 x 4096 NV12 frame whose 2x2 blocks hold every (U, V) pair with all 256 Y values: every triple once."""
    cv2 = pytest.importorskip("cv2")
    n = np.arange(1 << 22, dtype=np.uint32)                         # block index; block = 4 pixels with one (U, V)
    k, j = n >> 6, n & 63                                            # (U, V) index, which 4 of the 256 Y values
    luma = np.empty((4096, 4096), np.uint8)
    y4 = (4 * j[:, None] + np.arange(4, dtype=np.uint32)).astype(np.uint8).reshape(2048, 2048, 2, 2)
    luma[:] = y4.transpose(0, 2, 1, 3).reshape(4096, 4096)
    chroma = np.stack([(k >> 8).astype(np.uint8), (k & 255).astype(np.uint8)], -1).reshape(2048, 4096)
    want = cv2.cvtColor(np.concatenate([luma, chroma]), cv2.COLOR_YUV2RGB_NV12)
    got = yuv_spec.nv12_to_rgb(luma, chroma, "bt601")
    assert np.array_equal(got, want)
    covered = luma.astype(np.uint32) | (np.repeat(np.repeat(k.reshape(2048, 2048), 2, 0), 2, 1) << 8)
    assert np.unique(covered).size == 1 << 24


@pytest.mark.parametrize("hw", [(2, 2), (480, 640), (36, 1282)])
def test_bt601_limited_is_opencv_on_random_frames(hw):
    cv2 = pytest.importorskip("cv2")
    h, w = hw
    nv = np.random.default_rng(h + w).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    luma, chroma = yuv_spec.split_packed(nv)
    assert np.array_equal(yuv_spec.nv12_to_rgb(luma, chroma, 0), cv2.cvtColor(nv, cv2.COLOR_YUV2RGB_NV12))


@pytest.mark.parametrize("cs", [0, 1, 2, 3])
def test_every_row_is_within_one_level_of_float64(cs):
    Y, U, V = _all_triples()
    got = yuv_spec.yuv_to_rgb(Y, U, V, cs).astype(np.int16)
    want = yuv_spec.yuv_to_rgb_float(Y, U, V, cs).astype(np.int16)
    assert np.abs(got - want).max() <= 1


@pytest.mark.parametrize("cs", [1, 2, 3])
def test_rows_two_to_four_are_the_rounded_exact_coefficients(cs):
    assert yuv_spec.COEFFS[cs][:5] == tuple(round(c * 2 ** 20) for c in yuv_spec.exact_coeffs(cs))


def test_rows_match_the_header():
    with open(os.path.join(ROOT, "include", "lwdetr_b200.h")) as f:
        hdr = f.read()
    for cs, name in enumerate(("BT601_LIMITED", "BT709_LIMITED", "BT601_FULL", "BT709_FULL")):
        line = next(l for l in hdr.splitlines() if l.strip().startswith("*   LWDETR_CSC_" + name))
        assert tuple(int(v) for v in line.split()[2:7]) == yuv_spec.COEFFS[cs][:5], name


@pytest.mark.parametrize("cs", [0, 1, 2, 3])
def test_anchor_values(cs):
    limited = cs < 2
    black, white = (16, 235) if limited else (0, 255)
    rgb = yuv_spec.yuv_to_rgb(np.array([black, white, 0 if limited else 128]), np.full(3, 128), np.full(3, 128), cs)
    assert rgb[0].tolist() == [0, 0, 0] and rgb[1].tolist() == [255, 255, 255]
    assert rgb[2].tolist() == ([0, 0, 0] if limited else [128, 128, 128])         # below black clamps; full-range mid-grey
    grey = yuv_spec.yuv_to_rgb(np.array([126]), np.array([128]), np.array([128]), cs)[0]
    assert len(set(grey.tolist())) == 1                                              # no chroma: R = G = B


def test_odd_frames_use_the_ceil_sized_chroma_plane():
    rng = np.random.default_rng(5)
    luma = rng.integers(0, 256, (5, 7), dtype=np.uint8)
    chroma = rng.integers(0, 256, (3, 8), dtype=np.uint8)
    got = yuv_spec.nv12_to_rgb(luma, chroma, "bt709")
    for y in range(5):
        for x in range(7):
            want = yuv_spec.yuv_to_rgb(luma[y, x], chroma[y >> 1, 2 * (x >> 1)], chroma[y >> 1, 2 * (x >> 1) + 1], 1)
            assert np.array_equal(got[y, x], want)
    with pytest.raises(AssertionError):
        yuv_spec.nv12_to_rgb(luma, chroma[:, :6], 1)


def test_struct_matches_the_header():
    """lwdetr_frame_nv12: two (pointer, int64 pitch) planes, five int32, natural alignment: 56 bytes."""
    S = capi.FrameNV12Struct
    assert ctypes.sizeof(S) == 56
    assert [S.luma_pitch.offset, S.chroma.offset, S.chroma_pitch.offset, S.height.offset, S.colorspace.offset] == [8, 16, 24, 32, 48]
    assert {"lwdetr_forward_frames_nv12", "lwdetr_resize_patches_nv12"} <= set(capi.exported_symbols())
    assert capi.COLORSPACES == yuv_spec.NAMES


def test_host_checks_reject_bad_nv12_descriptors_without_a_gpu():
    fr = (capi.FrameNV12Struct * 1)()
    norm = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    dummy = ctypes.c_void_p(256)                                  # never dereferenced: every call below is rejected

    def call(h=64, w=64, lp=64, cp=64, dh=64, dw=64, cs=0, luma=256, chroma=512, H=128, W=128):
        d = fr[0]
        d.luma, d.luma_pitch, d.chroma, d.chroma_pitch = luma, lp, chroma, cp
        d.height, d.width, d.dst_h, d.dst_w, d.colorspace = h, w, dh, dw, cs
        rc = capi.lib().lwdetr_resize_patches_nv12(capi.F16, ctypes.cast(fr, ctypes.c_void_p), 1, H, W, ctypes.cast(norm, ctypes.c_void_p),
                                                   ctypes.cast(norm, ctypes.c_void_p), dummy, None, None)
        return rc, capi.lib().lwdetr_last_error().decode()

    for kw, msg in ((dict(luma=None), "null luma"), (dict(chroma=None), "null chroma"), (dict(h=4), "[8, 8192]"),
                    (dict(w=9000, lp=9000, cp=9000), "[8, 8192]"), (dict(lp=63), "luma_pitch 63"),
                    (dict(w=63, lp=63, cp=63), "chroma_pitch 63 is smaller than 2 * ceil(width / 2) = 64"),
                    (dict(cs=4), "unknown colorspace 4"), (dict(cs=-1), "unknown colorspace -1"),
                    (dict(dh=192), "run size 128x128"), (dict(dw=0), "run size 128x128"),
                    (dict(h=2064, dh=128), "factor above 16")):
        rc, err = call(**kw)
        assert rc != 0 and msg in err and err.startswith("lwdetr_resize_patches_nv12: frame 0"), (kw, err)
    rc, err = call(W=100)
    assert rc != 0 and "multiples of 64" in err
    rc, err = capi.lib().lwdetr_forward_frames_nv12(None, None, None, None, 1, 128, 128, None, None, None, None, None), None
    assert rc != 0 and "lwdetr_forward_frames_nv12: null pointer" in capi.lib().lwdetr_last_error().decode()


def test_python_rejections():
    u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="h and w even"):
        capi.Frames([u8(16, 8)], colorspace="bt601")                    # 16 rows are no 3h/2
    with pytest.raises(RuntimeError, match="h and w even"):
        capi.Frames(u8(2, 96, 63), colorspace="bt601")
    with pytest.raises(RuntimeError, match="h and w even"):
        capi.Frames([u8(97, 64)], colorspace="bt601")
    with pytest.raises(RuntimeError, match="not a mix"):
        capi.Frames([u8(16, 16, 3), u8(24, 16)], colorspace="bt601")
    with pytest.raises(RuntimeError, match="not a mix"):
        capi.Frames([(u8(16, 16), u8(8, 16)), u8(16, 16, 3)])
    with pytest.raises(RuntimeError, match="need colorspace"):
        capi.Frames([u8(24, 16)])
    with pytest.raises(RuntimeError, match="unknown colorspace 'bt2020'"):
        capi.Frames([u8(24, 16)], colorspace="bt2020")
    with pytest.raises(RuntimeError, match="2 colorspaces for 1 frames"):
        capi.Frames([u8(24, 16)], colorspace=["bt601", "bt709"])
    with pytest.raises(RuntimeError, match="NV12 frames only"):
        capi.Frames([u8(16, 16, 3)], colorspace="bt709")
    with pytest.raises(RuntimeError, match="CUDA"):
        capi.Frames([u8(24, 16)], colorspace="bt709")                  # well formed, but on the host
