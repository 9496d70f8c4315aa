"""CPU tests of the drawing contract (tools/annotate_spec.py, include/lwdetr_b200.h): outlines, fills, clipping, invalid
boxes, label placement at the four edges, cv2.rectangle at thickness 1, polygon fills against the zones' membership,
pixelation against a direct block mean, the RGB -> YUV table against the existing YUV -> RGB rows, the font header, and the
C ABI's refusals that need no device."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import annotate_spec as an  # noqa: E402
import yuv_spec  # noqa: E402
import zone_spec  # noqa: E402


def draw(a, img, boxes, labels=None, scores=None, **kw):
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    n = len(boxes)
    labels = np.zeros(n, np.int32) if labels is None else np.asarray(labels, np.int32)
    scores = np.ones(n, np.float32) if scores is None else np.asarray(scores, np.float32)
    return a.draw_rgb(img, scores=scores, labels=labels, boxes=boxes, **kw)


def test_outline_fill_and_clip():
    a = an.Annotator(4, label=0, thickness=3, box_fill_alpha=256, palette=[(10, 20, 30)])
    img = np.zeros((40, 50, 3), np.uint8)
    draw(a, img, [[5.7, 6.2, 20.9, 30.0]])
    want = np.zeros((40, 50), bool)
    want[6:30, 5:20] = True
    assert (img.any(-1) == want).all()
    assert (img[want] == (10, 20, 30)).all()
    a2 = an.Annotator(4, label=0, thickness=3)
    img = np.zeros((40, 50, 3), np.uint8)
    draw(a2, img, [[-10, -5, 30.5, 100]])                     # clamped to the frame: [0, 30) x [0, 40)
    ring = np.zeros((40, 50), bool)
    ring[0:40, 0:30] = True
    ring[3:37, 3:27] = False
    assert (img.any(-1) == ring).all()


@pytest.mark.parametrize("box", [[5, 5, 5, 9], [5, 5, 9, 5.5], [np.nan, 1, 4, 4], [1, 1, np.inf, 4], [60, 0, 70, 5], [-9, 3, -1, 9]])
def test_boxes_not_drawn(box):
    a = an.Annotator(4)
    img = np.full((30, 50, 3), 7, np.uint8)
    draw(a, img, [box])
    assert (img == 7).all()


def test_threshold_and_count():
    a = an.Annotator(4, label=0)
    img = np.zeros((30, 30, 3), np.uint8)
    draw(a, img, [[1, 1, 9, 9], [12, 12, 20, 20], [22, 22, 28, 28]], scores=[0.2, 0.6, 0.9], threshold=0.5, count=2)
    assert not img[1:9, 1:9].any() and img[12:20, 12:20].any() and not img[22:28, 22:28].any()


def test_outline_equals_cv2_rectangle():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    a = an.Annotator(8, label=0, thickness=1)
    for _ in range(20):
        h, w = rng.integers(10, 60, 2)
        x0, x1 = sorted(rng.integers(0, w + 1, 2))
        y0, y1 = sorted(rng.integers(0, h + 1, 2))
        if x1 == x0 or y1 == y0:
            continue
        lab = int(rng.integers(0, 8))
        base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        got = draw(a, base.copy(), [[x0, y0, x1, y1]], labels=[lab])
        want = base.copy()
        cv2.rectangle(want, (int(x0), int(y0)), (int(x1) - 1, int(y1) - 1), tuple(int(v) for v in a.colour(lab)), 1)
        assert np.array_equal(got, want)


def test_label_placement_at_the_edges():
    s = 2
    a = an.Annotator(4, names=["cat"], text_scale=s, label=an.LABEL_NAME, thickness=1)
    h, w = 60, 80
    tw, th = 3 * 6 * s, 8 * s
    cases = {                                   # box -> expected background rectangle (x0, y0, x1, y1), clipped
        "above": ([10, 30, 40, 50], (10, 30 - th, 10 + tw, 30)),
        "top edge, inside": ([10, 5, 40, 50], (10, 5, 10 + tw, 5 + th)),
        "right edge, clipped": ([70, 30, 80, 50], (70, 30 - th, 80, 30)),
        "left edge": ([0, 30, 40, 50], (0, 30 - th, tw, 30)),
        "bottom edge, clipped": ([10, 55, 40, 60], (10, 55 - th, 10 + tw, 55)),
        "bottom row inside": ([10, 0, 40, 60], (10, 0, 10 + tw, th)),
    }
    for name, (box, (x0, y0, x1, y1)) in cases.items():
        prims = a.primitives(h, w, scores=np.ones(1, np.float32), labels=np.zeros(1, np.int32), boxes=np.array([box], np.float32))
        bg, glyphs = prims[-2], prims[-1]
        assert bg["kind"] == "fill" and glyphs["kind"] == "text" and glyphs["text"] == "cat", name
        assert bg["box"] == (x0, y0, x1, y1), (name, bg["box"])
        img = np.zeros((h, w, 3), np.uint8)
        draw(a, img, [box])
        assert (img[y0:y1, x0:x1].reshape(-1, 3) != 0).any(1).all(), name


def test_label_text_and_colour():
    assert an.label_text(7, "person", 0, 12, np.float32(0.875)) == "person #12 0.88"
    assert an.label_text(7, "", 5, None, np.float32(1.0)) == "5 1.00"
    assert an.label_text(an.LABEL_SCORE, "x", 1, 3, np.float32(-0.2)) == "0.00"
    assert an.label_text(an.LABEL_ID, "x", 1, None, 0.5) == ""
    assert an.text_colour((255, 255, 255)) == (0, 0, 0) and an.text_colour((0, 0, 128)) == (255, 255, 255)


def zones_inside(poly, h, w):
    """Which pixel centres the zones count inside polygon `poly`: a track per pixel, its box's bottom-centre anchor (the
    default zone anchor) at the pixel centre, through one zone_spec.Stream update.  bool [h, w]."""
    ys, xs = np.mgrid[0:h, 0:w]
    boxes = np.stack([xs, ys - 0.5, xs + 1, ys + 0.5], -1).reshape(-1, 4).astype(np.float32)
    st = zone_spec.Stream(zone_spec.params(num_classes=1, capacity=h * w))
    st.set((), [poly])
    inside, occupancy, _ = st.update(np.arange(1, h * w + 1, dtype=np.int32), np.zeros(h * w, np.int32), boxes, h * w)
    assert occupancy[0] == (inside & 1).sum()
    return (inside & 1).astype(bool).reshape(h, w)


def test_polygon_fill_is_what_zones_count():
    rng = np.random.default_rng(1)
    h, w = 40, 50
    for poly in (zone_spec.star(25, 20, 18, 7, 5), rng.uniform(-5, 55, (9, 2)), [(5, 5), (45, 5), (45, 5.5), (5, 35)]):
        poly = np.asarray(poly, np.float64)
        a = an.Annotator(1, zone_fill_alpha=256, label=0, zone_thickness=1, palette=[(255, 0, 0)])
        img = np.zeros((h, w, 3), np.uint8)
        a.draw_rgb(img, scores=np.zeros(0, np.float32), labels=np.zeros(0, np.int32), boxes=np.zeros((0, 4), np.float32),
                   geometry=(np.zeros((0, 4)), [poly]), line_totals=[])
        prims = a.primitives(h, w, scores=np.zeros(0, np.float32), labels=np.zeros(0, np.int32), boxes=np.zeros((0, 4), np.float32),
                             geometry=(np.zeros((0, 4)), [poly]), line_totals=[])
        edges = np.zeros((h, w), bool)
        for q in prims:
            if q["kind"] == "seg":
                edges |= a.coverage(q, h, w)
        want = zones_inside(poly, h, w)
        assert want.any() and (~edges).any()
        assert np.array_equal(img[..., 0][~edges] == 255, want[~edges])       # off the outline: filled iff counted inside


def test_segment_rule():
    xs, ys = np.meshgrid(np.arange(20), np.arange(20))
    cov = an.segment_covers(xs, ys, (2.0, 10.0, 17.0, 10.0), 1.0)
    assert cov[9:11, 2:17].all() and not cov[8].any() and not cov[11].any()
    assert cov[9, 1] and not cov[9, 0]                         # round cap: centre (1.5, 9.5) is sqrt(0.5) from the end


def test_pixelation_is_block_mean():
    rng = np.random.default_rng(2)
    h, w, P = 37, 53, 8
    plane = rng.integers(0, 256, (h, w)).astype(np.uint8)
    cov = np.zeros((h, w), bool)
    cov[3:30, 5:50] = True
    cov[20:37, 40:53] = True
    got = an.pixelate(plane, cov, P)
    want = plane.copy()
    for by in range(0, h, P):
        for bx in range(0, w, P):
            m = cov[by:by + P, bx:bx + P]
            if m.any():
                blk = want[by:by + P, bx:bx + P]
                s, n = int(plane[by:by + P, bx:bx + P][m].astype(np.int64).sum()), int(m.sum())
                blk[m] = (s + n // 2) // n
    assert np.array_equal(got, want)


@pytest.mark.parametrize("cs", [0, 1, 2, 3])
def test_palette_yuv_round_trip(cs):
    rng = np.random.default_rng(cs)
    cols = np.concatenate([an.DEFAULT_PALETTE, rng.integers(0, 256, (500, 3)).astype(np.uint8),
                           np.array([(0, 0, 0), (255, 255, 255), (255, 0, 0), (0, 255, 0), (0, 0, 255)], np.uint8)])
    yuv = an.rgb_to_yuv(cols, cs)
    back = yuv_spec.yuv_to_rgb(yuv[:, 0], yuv[:, 1], yuv[:, 2], cs)
    assert np.abs(back.astype(int) - cols.astype(int)).max() <= 2


def test_font_header():
    assert an.FONT.shape == (95, 7) and an.FONT.max() < 32
    assert an.FONT[0].sum() == 0 and all(an.FONT[i].any() for i in range(1, 95))
    assert len({an.FONT[i].tobytes() for i in range(95)}) == 95


def test_nv12_chroma_weight():
    a = an.Annotator(4, label=0, thickness=32, palette=[(200, 40, 40)])   # the outline covers the box: one primitive
    luma = np.full((8, 8), 100, np.uint8)
    chroma = np.full((4, 8), 128, np.uint8)
    a.draw_nv12(luma, chroma, 0, scores=np.ones(1, np.float32), labels=np.zeros(1, np.int32), boxes=np.array([[1, 1, 4, 4]], np.float32))
    y, u, v = an.rgb_to_yuv(np.array([200, 40, 40], np.uint8), 0)
    assert (luma[1:4, 1:4] == y).all() and (luma[0] == 100).all()
    assert chroma[0, 0] == an.blend(128, u, (256 * 1 + 2) >> 2)       # one of its four pixels covered
    assert chroma[0, 2] == an.blend(128, u, (256 * 2 + 2) >> 2) and chroma[0, 3] == an.blend(128, v, (256 * 2 + 2) >> 2)
    assert chroma[1, 2] == u and chroma[1, 3] == v                    # all four
    assert (chroma[2:, 4:] == 128).all()


def test_options_validation_spec():
    with pytest.raises(ValueError):
        an.options(privacy_block=3)
    with pytest.raises(ValueError):
        an.options(thickness=33)
    with pytest.raises(ValueError):
        an.Annotator(4, names=["x" * 32])


def test_c_abi_refusals_without_a_device():
    from b200 import capi
    lib = capi.lib()
    out = ctypes.c_void_p()
    assert lib.lwdetr_annotator_create(0, ctypes.byref(out)) != 0
    assert b"num_classes" in lib.lwdetr_last_error()
    assert lib.lwdetr_annotator_create(1025, ctypes.byref(out)) != 0
    assert lib.lwdetr_annotator_set_option(None, b"thickness", 2) != 0
    assert b"null pointer" in lib.lwdetr_last_error()
    assert lib.lwdetr_annotator_set_names(None, b"a") != 0
    assert lib.lwdetr_annotator_set_palette(None, None, 1) != 0
    assert lib.lwdetr_annotate(None, None, 1, None, None, None, None, None, 1, 0.0, None, None, None, None) != 0
    assert lib.lwdetr_annotate_nv12(None, None, 1, None, None, None, None, None, 1, 0.0, None, None, None, None) != 0
    lib.lwdetr_annotator_destroy(None)
