"""Tiled detection (b200.config.tile_views, lwdetr_tile_merge in include/lwdetr_b200.h), restated in numpy for the tests.

views(): the view geometry, written independently of the planner.  merge(): the cross-view merge in numpy float32 with the
kernel's operation order: box + (x0, y0, x0, y0) in one fp32 add per coordinate; candidates sorted by score descending, ties
to the lower flat index view * k + rank; greedy class-aware NMS where only KEPT candidates suppress, with
  ix = max(0, min(ax2, bx2) - max(ax1, bx1)), iy likewise, inter = ix * iy, area = max(0, x2 - x1) * max(0, y2 - y1),
  iou: inter > thr * ((area_a + area_b) - inter),  ios: inter > thr * min(area_a, area_b),
each operation rounded to float32 on its own (numpy does not fuse), max / min as fmax / fmin (a NaN operand yields the other
one, as CUDA's fmaxf / fminf); a box whose area is not > 0 never suppresses and is never suppressed.
"""
import numpy as np


def axis_starts(n, t, overlap):
    s = t - int(overlap * t + 0.5)
    if n <= t:
        return [0]
    raw = list(range(0, n - t, s)) + [n - t]        # p + t < n  <=>  p < n - t
    return sorted({p - p % 2 for p in raw})


def views(shapes, tile, run, overlap=0.2, full_frame=True):
    """(frame, y0, x0, ch, cw, dst_h, dst_w) of every view: tile = (th, tw), run = (H, W)."""
    out = []
    for f, (h, w) in enumerate(shapes):
        ch, cw = min(tile[0], h), min(tile[1], w)
        dst = [R if c == t else min(max(int(np.floor(c * R / t + 0.5)), 1), R) for c, t, R in ((ch, tile[0], run[0]), (cw, tile[1], run[1]))]
        out += [(f, y0, x0, ch, cw, dst[0], dst[1]) for y0 in axis_starts(h, tile[0], overlap) for x0 in axis_starts(w, tile[1], overlap)]
        if full_frame:
            out.append((f, 0, 0, h, w, run[0], run[1]))
    return out


def _overlaps(a, aa, b, ab, thr, metric):
    """Does kept box a (area aa) suppress each of the boxes b [n, 4] (areas ab [n])?"""
    f32 = np.float32
    ix = np.fmax(f32(0), np.fmin(a[2], b[:, 2]) - np.fmax(a[0], b[:, 0]))
    iy = np.fmax(f32(0), np.fmin(a[3], b[:, 3]) - np.fmax(a[1], b[:, 1]))
    inter = ix * iy
    den = (aa + ab) - inter if metric == "iou" else np.fmin(aa, ab)
    with np.errstate(invalid="ignore"):
        return (inter > f32(thr) * den) & (aa > 0) & (ab > 0)


def area(b):
    f32 = np.float32
    return np.fmax(f32(0), b[..., 2] - b[..., 0]) * np.fmax(f32(0), b[..., 3] - b[..., 1])


def merge(scores, labels, boxes, tviews, num_frames, score_threshold=0.0, iou_threshold=0.5, metric="ios", max_det=300):
    """scores float32 [V, k], labels int [V, k], boxes float32 [V, k, 4] (view crop pixels), tviews: (frame, x0, y0) per view
    -> (scores [F, max_det] float32, labels [F, max_det] int32, boxes [F, max_det, 4] float32, counts [F] int32), unused
    slots 0 / -1 / zero box."""
    scores = np.asarray(scores, dtype=np.float32)
    labels = np.asarray(labels).astype(np.int32)
    boxes = np.asarray(boxes, dtype=np.float32)
    V, k = scores.shape
    f32 = np.float32
    o_s = np.zeros((num_frames, max_det), np.float32)
    o_l = np.full((num_frames, max_det), -1, np.int32)
    o_b = np.zeros((num_frames, max_det, 4), np.float32)
    counts = np.zeros(num_frames, np.int32)
    for f in range(num_frames):
        vs = [v for v in range(V) if tviews[v][0] == f]
        if not vs:
            continue
        s = scores[vs].reshape(-1)
        lab = labels[vs].reshape(-1)
        off = np.array([[tviews[v][1], tviews[v][2], tviews[v][1], tviews[v][2]] for v in vs], np.float32)
        b = (boxes[vs] + off[:, None, :]).reshape(-1, 4)
        flat = np.arange(s.size)
        keep_mask = s >= f32(score_threshold)
        idx = flat[keep_mask]
        sk = s[idx]
        order = idx[np.lexsort((idx, -sk.astype(np.float64)))]   # score descending (-0.0 == +0.0), then lower flat index
        s, lab, b = s[order], lab[order], b[order]
        ar = area(b)
        alive = np.ones(len(order), bool)
        kept = []
        for i in range(len(order)):
            if not alive[i]:
                continue
            kept.append(i)
            if len(kept) == max_det:
                break
            rest = slice(i + 1, None)
            same = lab[rest] == lab[i]
            alive[rest] &= ~(same & _overlaps(b[i], ar[i], b[rest], ar[rest], iou_threshold, metric))
        n = len(kept)
        counts[f] = n
        o_s[f, :n], o_l[f, :n], o_b[f, :n] = s[kept], lab[kept], b[kept]
    return o_s, o_l, o_b, counts
