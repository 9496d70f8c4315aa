"""CPU tests of tiled detection: the view planner (b200.config.tile_views) and the merge's specification
(tools/tile_spec.py) against torchvision's batched_nms (IoU) and a float64 loop (IoS)."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tile_spec  # noqa: E402
from b200.config import CONFIGS, tile_views  # noqa: E402

CFG = CONFIGS["small"]


# ----------------------------------------------------------------------------------------------- planner
@pytest.mark.parametrize("shape, rows, cols", [((1080, 1920), [0, 440], [0, 512, 1024, 1280]),
                                               ((2160, 3840), [0, 512, 1024, 1520], [0, 512, 1024, 1536, 2048, 2560, 3072, 3200])])
def test_grids_of_1080p_and_4k(shape, rows, cols):
    (H, W), views = tile_views(CFG, [shape], tile=640, overlap=0.2)
    assert (H, W) == (640, 640)
    assert len(views) == len(rows) * len(cols) + 1
    assert views[:-1] == [(0, y0, x0, 640, 640, 640, 640) for y0 in rows for x0 in cols]     # row-major, 1:1
    assert views[-1] == (0, 0, 0, shape[0], shape[1], 640, 640)                               # the full view last
    assert views == tile_spec.views([shape], (640, 640), (640, 640), 0.2)


SHAPES = [(1080, 1920), (2160, 3840), (1081, 1919), (721, 1283), (480, 640), (300, 200), (641, 1301), (8, 8), (4321, 777)]


@pytest.mark.parametrize("tile, overlap, size", [(None, 0.2, None), (640, 0.0, None), ((512, 768), 0.25, (448, 768)),
                                                 (333, 0.5, None), (1000, 0.1, (512, 512)), ((96, 130), 0.3, (320, 320))])
def test_views_cover_each_frame_with_even_starts(tile, overlap, size):
    (H, W), views = tile_views(CFG, SHAPES, tile=tile, overlap=overlap, size=size, per_view=1)
    th, tw = (H, W) if tile is None else ((tile, tile) if isinstance(tile, int) else tile)
    assert views == tile_spec.views(SHAPES, (th, tw), (H, W), overlap)
    assert [v[0] for v in views] == sorted(v[0] for v in views)                                 # frames in order
    for f, (h, w) in enumerate(SHAPES):
        mine = [v for v in views if v[0] == f]
        assert mine[-1] == (f, 0, 0, h, w, H, W)
        tiles = mine[:-1]
        assert [(v[1], v[2]) for v in tiles] == sorted((v[1], v[2]) for v in tiles)              # row-major
        cover = np.zeros((h, w), bool)
        for _, y0, x0, ch, cw, dh, dw in tiles:
            assert y0 % 2 == 0 and x0 % 2 == 0
            assert 0 <= y0 and y0 + ch <= h and 0 <= x0 and x0 + cw <= w
            assert (ch, cw) == (min(th, h), min(tw, w))
            for c, t, R, d in ((ch, th, H, dh), (cw, tw, W, dw)):
                assert d == (R if c == t else min(max(int(np.floor(c * R / t + 0.5)), 1), R))
            cover[y0:y0 + ch, x0:x0 + cw] = True
        # only the documented strip may stay uncovered: the last row / column when n - t is odd, and only if the overlap
        # is at least one pixel (otherwise rounding starts down may open a one-pixel gap between tiles)
        if int(overlap * th + 0.5) >= 1 and int(overlap * tw + 0.5) >= 1:
            ok_rows = h - 1 if h > th and (h - th) % 2 else h
            ok_cols = w - 1 if w > tw and (w - tw) % 2 else w
            assert cover[:ok_rows, :ok_cols].all(), (f, h, w)


def test_frame_smaller_than_the_tile_is_one_partial_view():
    (H, W), views = tile_views(CFG, [(480, 640), (300, 1500)], tile=(800, 1000), size=(640, 640), full_frame=False)
    # 480 / 800 * 640 = 384; 640 / 1000 * 640 = 409.6 -> 410; 300 / 800 * 640 = 240
    assert views == [(0, 0, 0, 480, 640, 384, 410), (1, 0, 0, 300, 1000, 240, 640), (1, 0, 500, 300, 1000, 240, 640)]


def test_out_of_range_parameters_raise():
    for kw, msg in ((dict(overlap=-0.1), "overlap"), (dict(overlap=0.6), "overlap"), (dict(tile=640 * 16 + 1), "above 16"),
                    (dict(tile=(100, 10241)), "above 16"), (dict(tile=0), "positive"), (dict(size=(600, 640)), "multiples of 64"),
                    (dict(tile=128, per_view=100), "16384 candidates"), (dict(tile=64, per_view=1, overlap=0.5), "2048 views")):
        with pytest.raises(RuntimeError, match=msg):
            tile_views(CFG, [(2160, 3840)], **kw)
    with pytest.raises(RuntimeError, match="above 16"):
        tile_views(CFG, [(6000, 6000)], size=(320, 320), tile=640)          # the full view would shrink 18.75x
    assert len(tile_views(CFG, [(6000, 6000)], size=(320, 320), tile=640, full_frame=False)[1]) == 12 * 12
    # a tile at exactly 16x the run size is accepted, but a 23-pixel partial crop of it goes to dst 1: 23x, rejected
    assert tile_views(CFG, [(6000, 6000)], size=(320, 320), tile=16 * 320, full_frame=False)[1][0][5:] == (320, 320)
    with pytest.raises(RuntimeError, match="crop goes to 1x320, a downscale factor above 16"):
        tile_views(CFG, [(23, 6000)], size=(320, 320), tile=16 * 320, full_frame=False)


# ----------------------------------------------------------------------------------------------- merge specification
def candidates(seed, V, k, ncls=4, span=300.0, wh=(8.0, 90.0), degenerate=0.0, ties=False):
    """Per-view postprocess-like output: scores [V, k] (distinct unless ties), labels, xyxy boxes in crop pixels."""
    rng = np.random.default_rng(seed)
    n = V * k
    if ties:
        scores = rng.integers(1, 6, n).astype(np.float32) / 8
    else:
        scores = ((rng.permutation(n) + 1) / (n + 1)).astype(np.float32)
    labels = rng.integers(0, ncls, n).astype(np.int32)
    cx, cy = rng.random(n) * span, rng.random(n) * span
    w, h = rng.uniform(*wh, n), rng.uniform(*wh, n)
    boxes = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], -1).astype(np.float32)
    if degenerate:
        d = rng.random(n) < degenerate
        boxes[d, 2] = boxes[d, 0] - rng.integers(0, 2, d.sum())           # zero or negative width
    return scores.reshape(V, k), labels.reshape(V, k), boxes.reshape(V, k, 4)


def random_views(seed, counts):
    rng = np.random.default_rng(seed)
    return [(f, int(rng.integers(0, 2000)) * 2, int(rng.integers(0, 1000)) * 2) for f, c in enumerate(counts) for _ in range(c)]


def _frame_boxes(boxes, views):
    off = np.array([[x0, y0, x0, y0] for _, x0, y0 in views], np.float32)
    return boxes + off[:, None, :]


def _drop_near_threshold(scores, labels, fboxes, views, thr, metric):
    """Sets the score of the later candidate of every same-frame, same-label pair whose float64 overlap lies within 1e-5
    (relative) of the threshold to -1 (below any threshold used here), so that rounding cannot decide a comparison."""
    scores = scores.copy()
    frames = np.repeat([v[0] for v in views], scores.shape[1])
    s, l, b = scores.reshape(-1), labels.reshape(-1), fboxes.reshape(-1, 4).astype(np.float64)
    area = np.maximum(0, b[:, 2] - b[:, 0]) * np.maximum(0, b[:, 3] - b[:, 1])
    ix = np.maximum(0, np.minimum(b[:, None, 2], b[None, :, 2]) - np.maximum(b[:, None, 0], b[None, :, 0]))
    iy = np.maximum(0, np.minimum(b[:, None, 3], b[None, :, 3]) - np.maximum(b[:, None, 1], b[None, :, 1]))
    inter = ix * iy
    den = area[:, None] + area[None, :] - inter if metric == "iou" else np.minimum(area[:, None], area[None, :])
    with np.errstate(invalid="ignore", divide="ignore"):
        r = inter / den
    near = (np.abs(r - thr) <= 1e-5 * thr) & (l[:, None] == l[None, :]) & (frames[:, None] == frames[None, :])
    i, j = np.nonzero(np.triu(near, 1))
    s[np.maximum(i, j)] = -1.0
    return s.reshape(scores.shape)


def _loop64(scores, labels, fboxes, views, F, thr, metric, max_det):
    """Greedy class-aware NMS in float64 by plain loops (score desc, ties to the lower flat index)."""
    out = []
    for f in range(F):
        vs = [v for v in range(len(views)) if views[v][0] == f]
        s = scores[vs].reshape(-1).astype(np.float64)
        l = labels[vs].reshape(-1)
        b = fboxes[vs].reshape(-1, 4).astype(np.float64)
        order = sorted((i for i in range(len(s)) if s[i] >= 0), key=lambda i: (-s[i], i))
        area = lambda x: max(0.0, x[2] - x[0]) * max(0.0, x[3] - x[1])
        kept = []
        for i in order:
            sup = False
            for j in kept:
                if l[j] != l[i] or area(b[j]) <= 0 or area(b[i]) <= 0:
                    continue
                inter = max(0.0, min(b[i][2], b[j][2]) - max(b[i][0], b[j][0])) * max(0.0, min(b[i][3], b[j][3]) - max(b[i][1], b[j][1]))
                den = area(b[i]) + area(b[j]) - inter if metric == "iou" else min(area(b[i]), area(b[j]))
                if inter > thr * den:
                    sup = True
                    break
            if not sup:
                kept.append(i)
                if len(kept) == max_det:
                    break
        out.append([(s[i], l[i], tuple(b[i])) for i in kept])
    return out


def _spec_as_lists(got):
    s, l, b, c = got
    return [[(float(s[f, i]), int(l[f, i]), tuple(float(x) for x in b[f, i])) for i in range(c[f])] for f in range(len(c))]


@pytest.mark.parametrize("seed, counts, k, thr, max_det", [(0, [3, 5], 40, 0.5, 300), (1, [1, 9, 2], 30, 0.3, 50),
                                                           (2, [4], 100, 0.7, 1000), (3, [2, 2], 64, 0.5, 5)])
def test_merge_iou_equals_torchvision_batched_nms(seed, counts, k, thr, max_det):
    torch = pytest.importorskip("torch")
    tv = pytest.importorskip("torchvision")
    views = random_views(seed, counts)
    scores, labels, boxes = candidates(seed, len(views), k, span=150.0)
    fboxes = _frame_boxes(boxes, views)
    scores = _drop_near_threshold(scores, labels, fboxes, views, thr, "iou")
    got = tile_spec.merge(scores, labels, boxes, views, len(counts), 0.0, thr, "iou", max_det)
    for f in range(len(counts)):
        vs = [v for v in range(len(views)) if views[v][0] == f]
        s, l, b = scores[vs].reshape(-1), labels[vs].reshape(-1), fboxes[vs].reshape(-1, 4)
        live = np.nonzero(s >= 0)[0]
        keep = tv.ops.batched_nms(torch.from_numpy(b[live]).double(), torch.from_numpy(s[live]).double(),
                                  torch.from_numpy(l[live]).long(), thr)[:max_det].numpy()
        idx = live[keep]
        n = int(got[3][f])
        assert n == len(idx) and n > 1
        assert np.array_equal(got[0][f, :n], s[idx]) and np.array_equal(got[1][f, :n], l[idx]) and np.array_equal(got[2][f, :n], b[idx])
        assert (got[0][f, n:] == 0).all() and (got[1][f, n:] == -1).all() and (got[2][f, n:] == 0).all()


@pytest.mark.parametrize("seed, counts, k, thr, max_det, degenerate", [(10, [3, 5], 40, 0.5, 300, 0.0), (11, [1, 9, 2], 30, 0.3, 50, 0.1),
                                                                       (12, [4], 100, 0.8, 1000, 0.0), (13, [2, 0, 2], 64, 0.5, 7, 0.05)])
def test_merge_ios_equals_a_float64_loop(seed, counts, k, thr, max_det, degenerate):
    views = random_views(seed, counts)
    scores, labels, boxes = candidates(seed, len(views), k, span=150.0, degenerate=degenerate)
    fboxes = _frame_boxes(boxes, views)
    scores = _drop_near_threshold(scores, labels, fboxes, views, thr, "ios")
    got = _spec_as_lists(tile_spec.merge(scores, labels, boxes, views, len(counts), 0.0, thr, "ios", max_det))
    want = _loop64(scores, labels, fboxes, views, len(counts), thr, "ios", max_det)
    assert [len(g) for g in got] == [len(w) for w in want]
    assert sum(len(g) for g in got) > 0
    for g, w in zip(got, want):
        assert g == [(np.float32(s), l, tuple(np.float32(x) for x in b)) for s, l, b in w]


def test_merge_keeps_ties_in_flat_order_and_ios_absorbs_cut_boxes():
    # two views of one frame; view 1 sits 100 px to the right.  A box cut at view 0's border (inside the whole-object box of
    # view 1) has IoU 0.4 with it but IoS 1: IoS merges the two, IoU keeps both.
    scores = np.array([[0.5, 0.9], [0.9, 0.1]], np.float32)
    labels = np.array([[1, 2], [2, 1]], np.int32)
    boxes = np.array([[[0, 0, 10, 10], [140, 0, 160, 50]], [[40, 0, 60, 50], [500, 500, 510, 510]]], np.float32)
    views = [(0, 0, 0), (0, 100, 0)]
    cut = np.array([[0, 0, 10, 10], [140, 0, 148, 50]], np.float32)
    s, l, b, c = tile_spec.merge(scores, labels, np.stack([cut, boxes[1]]), views, 1, 0.0, 0.5, "ios", 10)
    # order: 0.9 (view 0 rank 1, flat 1) before 0.9 (view 1 rank 0, flat 2); flat 2 (label 2) is not inside flat 1, flat 1
    # is inside flat 2: with flat 1 first, IoS(flat 1, flat 2) = 400 / 400 = 1 -> flat 2 suppressed
    assert c[0] == 3 and list(l[0, :3]) == [2, 1, 1] and list(b[0, 0]) == [140, 0, 148, 50]
    s, l, b, c = tile_spec.merge(scores, labels, np.stack([cut, boxes[1]]), views, 1, 0.0, 0.5, "iou", 10)
    assert c[0] == 4                                                         # IoU 400 / 1000 = 0.4: both kept


def test_tile_merge_symbol_is_declared():
    from b200 import capi
    with open(os.path.join(ROOT, "include", "lwdetr_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"LWDETR_API\s+int\s+lwdetr_tile_merge\s*\(", hdr)
    assert "lwdetr_tile_merge" in capi.exported_symbols()
    assert re.search(r"LWDETR_TILE_IOU\s*=\s*0,\s*LWDETR_TILE_IOS\s*=\s*1", hdr)
    assert hasattr(capi.lib(), "lwdetr_tile_merge")
