"""CPU tests of the detection-crop contract (tools/crop_spec.py, include/lwdetr_b200.h lwdetr_crops): the bilinear filter
within one level of cv2.resize(INTER_LINEAR), the antialias filter equal to the frame path's resize, the crop rectangle's edge
cases, NV12 crops at odd offsets, the selection order, and the new symbols in the cross-compiled library."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import crop_spec  # noqa: E402
import resize_spec  # noqa: E402
import yuv_spec  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _sizes(rng, n):
    """Random crop sides from 1 to 600 px, biased to small ones, with every 1-px combination."""
    out = [(1, 1), (1, 37), (53, 1), (2, 2)]
    while len(out) < n:
        out.append(tuple(int(v) for v in np.minimum(np.exp(rng.uniform(0, np.log(600), 2)).astype(int) + 1, 600)))
    return out


@pytest.mark.parametrize("dst", [(256, 128), (64, 32), (300, 700)])
def test_bilinear_within_one_level_of_cv2(dst):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(dst[0] + dst[1])
    diff_share = []
    for h, w in _sizes(rng, 80):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        got = resize_spec.round_levels(crop_spec.resize_levels(img, dst[0], dst[1], "bilinear"))
        want = cv2.resize(img, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
        d = np.abs(got.astype(int) - want.astype(int))
        assert d.max() <= 1, ((h, w), d.max())
        diff_share.append((d > 0).mean())
    assert max(diff_share) < 0.2, max(diff_share)
    print("bilinear vs cv2 at %s: mean share of one-level differences %.3f, worst %.3f" % (dst, np.mean(diff_share), max(diff_share)))


def test_antialias_equals_the_frame_resize():
    rng = np.random.default_rng(3)
    for h, w in _sizes(rng, 30) + [(1080, 1920)]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for dst in ((256, 128), (8, 8)):
            got = resize_spec.round_levels(crop_spec.resize_levels(img, dst[0], dst[1], "antialias"))
            assert np.array_equal(got, resize_spec.resize_u8(img, *dst)), (h, w, dst)


def test_crop_rect_edge_cases():
    r = crop_spec.crop_rect
    assert r([10.7, 5.2, 20.9, 30.0], 100, 200) == (10, 5, 20, 30)            # fractional: truncation of tlbr.astype(int)
    assert r([-5.5, -1.0, 3.2, 4.9], 100, 200) == (0, 0, 3, 4)                 # negative start clamps to 0
    assert r([190.0, 90.0, 250.0, 150.0], 100, 200) == (190, 90, 200, 100)     # past the frame clamps to the side
    assert r([-50.0, -50.0, -1.0, -2.0], 100, 200) is None                      # entirely outside, before
    assert r([200.0, 10.0, 260.0, 20.0], 100, 200) is None                      # entirely outside, after
    assert r([10.0, 10.0, 10.9, 30.0], 100, 200) is None                        # degenerate after truncation
    assert r([10.0, 10.0, 5.0, 30.0], 100, 200) is None                         # inverted
    for bad in (np.nan, np.inf, -np.inf):
        for i in range(4):
            b = [1.0, 1.0, 50.0, 50.0]
            b[i] = bad
            assert r(b, 100, 200) is None
    assert r([-1e30, -1e30, 1e30, 1e30], 100, 200) == (0, 0, 200, 100)


def test_invalid_crops_are_zeros_with_flag_zero():
    rng = np.random.default_rng(4)
    frame = rng.integers(0, 256, (40, 60, 3), dtype=np.uint8)
    boxes = [[1, 1, 20, 30], [np.nan, 0, 5, 5], [70, 0, 80, 10], [3, 3, 9, 9]]
    vals, u8, _, valid = crop_spec.crops([frame], boxes, [0, 0, 0, 1], (16, 8), "bilinear", MEAN, STD)
    assert list(valid) == [True, False, False, False]
    assert not vals[1:].any() and not u8[1:].any()


@pytest.mark.parametrize("filter", crop_spec.FILTERS)
def test_nv12_crops_equal_rgb_crops_of_the_converted_frame_at_odd_offsets(filter):
    rng = np.random.default_rng(5)
    h, w = 75, 123
    luma = rng.integers(0, 256, (h, w), dtype=np.uint8)
    chroma = rng.integers(0, 256, ((h + 1) // 2, 2 * ((w + 1) // 2)), dtype=np.uint8)
    rgb = crop_spec.nv12_frames([(luma, chroma)], ["bt709"])[0]
    assert np.array_equal(rgb, yuv_spec.nv12_to_rgb(luma, chroma, "bt709"))
    for x0, y0, x1, y1 in ((3, 5, 40, 61), (1, 1, 2, 2), (99, 7, 123, 75)):
        got = crop_spec.crop_levels(rgb, [x0 + 0.5, y0 + 0.25, x1 + 0.9, y1], (16, 8), filter)
        # a crop of the converted frame: odd offsets take the chroma of the whole frame, not of a re-based tile
        want = crop_spec.resize_levels(rgb[y0:y1, x0:x1], 16, 8, filter)
        assert np.array_equal(got, want)


def test_selection_order_and_count():
    scores = np.array([[0.9, 0.2, 0.7, 0.8], [0.1, 0.95, 0.6, 0.5]], np.float32)
    boxes = np.array([[[0, 0, 10, 10], [0, 0, 5, 5], [50, 50, 60, 60], [1, 1, np.nan, 5]],
                      [[0, 0, 3, 3], [2, 2, 2.5, 9], [4, 4, 8, 8], [5, 5, 9, 9]]], np.float32)
    sel = crop_spec.select(scores, boxes, [(40, 40), (40, 40)], 0.5)
    # frame 0: entry 0 kept, 1 below, 2 outside the 40x40 frame, 3 NaN; frame 1: 1 degenerate, 2 kept, 3 not > 0.5
    assert [(b, e) for b, e, _ in sel] == [(0, 0), (1, 6)]
    assert [e for _, e, _ in crop_spec.select(scores, boxes, [(80, 80), (40, 40)], 0.0)] == [0, 1, 2, 4, 6, 7]


def test_new_symbols_are_in_the_built_library():
    lib = os.path.join(ROOT, "lw-detr_b200", "lib", "liblwdetr_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    import subprocess
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for s in ("lwdetr_crops", "lwdetr_crops_nv12", "lwdetr_crop_select", "lwdetr_scatter_rows"):
        assert (" T %s\n" % s) in out, s
