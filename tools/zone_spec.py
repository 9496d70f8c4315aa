"""Line crossings and zone occupancy per camera stream (lwdetr_zones_* in include/lwdetr_b200.h), restated in numpy for the
tests: what DeepStream's nvdsanalytics and supervision's LineZone / PolygonZone compute after the tracker, on the tracker's
own outputs (ids, labels, xyxy boxes in frame pixels, counts).

Everything is float64 with each operation rounded on its own (numpy does not fuse), in the order the header fixes.  The
geometry tests are vectorised over the present tracks; elementwise numpy arithmetic rounds each operation exactly as the
kernel's __dadd_rn / __dmul_rn / __ddiv_rn do, so the two agree bit for bit.
"""
import numpy as np

MAX_LINES, MAX_POLYGONS, MAX_POLY_VERTICES, MAX_VERTICES = 32, 32, 256, 2048
MAX_CAPACITY, MAX_CLASSES = 4096, 1024
LINE_IN, LINE_OUT, ZONE_ENTER, ZONE_EXIT, ZONE_FORGET = 1, 2, 3, 4, 5

# anchors of a box: index 3 * row + column, rows top / centre / bottom, columns left / centre / right
TOP_LEFT, TOP_CENTER, TOP_RIGHT, CENTER_LEFT, CENTER, CENTER_RIGHT, BOTTOM_LEFT, BOTTOM_CENTER, BOTTOM_RIGHT = range(9)
CORNERS = (1 << TOP_LEFT) | (1 << TOP_RIGHT) | (1 << BOTTOM_LEFT) | (1 << BOTTOM_RIGHT)

DEFAULTS = dict(num_classes=91, capacity=1024, forget_after=30, zone_anchor=BOTTOM_CENTER, line_anchors=CORNERS)


def params(**kw):
    """The parameter block with lwdetr_zones_params_default's values, validated as lwdetr_zones_create does."""
    bad = set(kw) - set(DEFAULTS)
    if bad:
        raise TypeError("unknown zone parameters: %s" % ", ".join(sorted(bad)))
    p = dict(DEFAULTS)
    p.update(kw)
    if not 1 <= p["num_classes"] <= MAX_CLASSES or not 1 <= p["capacity"] <= MAX_CAPACITY or p["forget_after"] < 0 \
            or not 0 <= p["zone_anchor"] < 9 or not 0 < p["line_anchors"] < 512:
        raise ValueError("zone parameters out of range: %s" % p)
    return p


def geometry(lines=(), polygons=()):
    """Validated geometry of one stream: (lines float64 [L, 4], polygons: list of float64 [n, 2]).  ValueError on more than
    32 lines or 32 polygons, a polygon outside 3..256 vertices, more than 2048 vertices, a non-finite coordinate or a
    zero-length line."""
    ln = np.asarray(lines, np.float64).reshape(-1, 4) if len(lines) else np.zeros((0, 4))
    if len(ln) > MAX_LINES:
        raise ValueError("at most %d lines, got %d" % (MAX_LINES, len(ln)))
    if not np.isfinite(ln).all():
        raise ValueError("line coordinates must be finite")
    if ((ln[:, 0] == ln[:, 2]) & (ln[:, 1] == ln[:, 3])).any():
        raise ValueError("a line has zero length")
    polys = [np.asarray(p, np.float64) for p in polygons]
    if len(polys) > MAX_POLYGONS:
        raise ValueError("at most %d polygons, got %d" % (MAX_POLYGONS, len(polys)))
    for p in polys:
        if p.ndim != 2 or p.shape[1] != 2 or not 3 <= len(p) <= MAX_POLY_VERTICES:
            raise ValueError("a polygon is [n, 2] with n in [3, %d], got %s" % (MAX_POLY_VERTICES, p.shape))
        if not np.isfinite(p).all():
            raise ValueError("polygon coordinates must be finite")
    if sum(len(p) for p in polys) > MAX_VERTICES:
        raise ValueError("at most %d vertices per stream" % MAX_VERTICES)
    return ln, polys


def anchors(boxes, which):
    """Anchor `which` (0..8) of fp32 xyxy boxes [n, 4], widened to float64: (x, y) arrays."""
    b = np.asarray(boxes, np.float32).astype(np.float64).reshape(-1, 4)
    row, col = divmod(which, 3)
    x = (b[:, 0], (b[:, 0] + b[:, 2]) * 0.5, b[:, 2])[col]
    y = (b[:, 1], (b[:, 1] + b[:, 3]) * 0.5, b[:, 3])[row]
    return x, y


def line_sides(boxes, line, mask):
    """Each box's decision for one line (ax, ay, bx, by): +1 when every anchor in `mask` has 0 <= t <= L2 and c > 0, -1 when
    every one has 0 <= t <= L2 and c < 0, else 0.  int8 [n]."""
    ax, ay, bx, by = (np.float64(v) for v in line)
    dx, dy = bx - ax, by - ay
    L2 = dx * dx + dy * dy
    n = len(boxes)
    pos, neg = np.ones(n, bool), np.ones(n, bool)
    for a in range(9):
        if mask >> a & 1:
            px, py = anchors(boxes, a)
            t = (px - ax) * dx + (py - ay) * dy
            c = dx * (py - ay) - dy * (px - ax)
            within = (t >= 0) & (t <= L2)
            pos &= within & (c > 0)
            neg &= within & (c < 0)
    return np.where(pos, 1, np.where(neg, -1, 0)).astype(np.int8)


def inside_polygon(px, py, poly):
    """Crossing-number (even-odd) rule in the header's form: for i = 0..n-1, j = (i + n - 1) % n, the point flips inside
    when (yi > py) != (yj > py) and px < (xj - xi) * (py - yi) / (yj - yi) + xi.  Points on edges get what this half-open
    rule gives.  bool [len(px)]."""
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    inside = np.zeros(px.shape, bool)
    n = len(poly)
    for i in range(n):
        xi, yi = poly[i]
        xj, yj = poly[(i + n - 1) % n]
        straddle = (yi > py) != (yj > py)
        with np.errstate(divide="ignore", invalid="ignore"):
            x = (xj - xi) * (py - yi) / (yj - yi) + xi
        inside ^= straddle & (px < x)
    return inside


class Stream:
    """One stream's geometry, records (one per track id) and counters."""

    def __init__(self, p):
        self.p = p
        self.lines, self.polys = geometry()
        self.reset()

    def _clear(self):
        nc = self.p["num_classes"] + 1
        self.records = {}
        self.overflow = 0
        self.line_counts = np.zeros((MAX_LINES, nc, 2), np.int64)
        self.entries = np.zeros((MAX_POLYGONS, nc), np.int64)

    def reset(self):
        """Frame back to 1; records, counters and overflow cleared; geometry kept."""
        self.frame = 1
        self._clear()

    def set(self, lines=(), polygons=()):
        """New geometry; the records and counters are cleared, the frame count goes on."""
        self.lines, self.polys = geometry(lines, polygons)
        self._clear()

    def update(self, ids, labels, boxes, count, max_out=None):
        """One frame: the tracker's ids int32 [max_out], labels int32, boxes fp32 [max_out, 4] and count ->
        (inside uint32 [max_out], occupancy int32 [32], events: list of (id, kind, index, label, dwell))."""
        ids = np.asarray(ids, np.int32)
        labels = np.asarray(labels, np.int32)
        boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
        max_out = len(ids) if max_out is None else max_out
        p, L, Z, frame = self.p, len(self.lines), len(self.polys), self.frame
        present, seen = [], set()
        for j in range(max(0, min(int(count), max_out))):
            i = int(ids[j])
            if i <= 0 or not np.isfinite(boxes[j]).all() or i in seen:
                continue
            seen.add(i)
            present.append(j)
        pb = boxes[present]
        sides = np.stack([line_sides(pb, self.lines[l], p["line_anchors"]) for l in range(L)], 1) if L else np.zeros((len(pb), 0), np.int8)
        zx, zy = anchors(pb, p["zone_anchor"])
        masks = np.zeros(len(pb), np.int64)
        for z in range(Z):
            masks |= inside_polygon(zx, zy, self.polys[z]).astype(np.int64) << z
        inside = np.zeros(max_out, np.uint32)
        occ = np.zeros(MAX_POLYGONS, np.int32)
        events = []
        free = p["capacity"] - len(self.records)
        other = p["num_classes"]
        for q, j in enumerate(present):
            tid, lab, m = int(ids[j]), int(labels[j]), int(masks[q])
            inside[j] = m
            for z in range(Z):
                occ[z] += m >> z & 1
            rec = self.records.get(tid)
            if rec is None:
                if free == 0:
                    self.overflow += 1
                    continue
                free -= 1
                rec = dict(label=lab, last_seen=frame, sides=np.zeros(MAX_LINES, np.int8), inside=0,
                           entry=np.zeros(MAX_POLYGONS, np.int32))
                self.records[tid] = rec
            col = lab if 0 <= lab < other else other
            for l in range(L):
                d = int(sides[q, l])
                if d == 0:
                    continue
                s = int(rec["sides"][l])
                if s != 0 and d != s:
                    kind = LINE_IN if d == 1 else LINE_OUT
                    self.line_counts[l, col, kind - LINE_IN] += 1
                    events.append((tid, kind, l, lab, 0))
                rec["sides"][l] = d
            for z in range(Z):
                now, was = m >> z & 1, rec["inside"] >> z & 1
                if now and not was:
                    rec["entry"][z] = frame
                    self.entries[z, col] += 1
                    events.append((tid, ZONE_ENTER, z, lab, 0))
                elif was and not now:
                    events.append((tid, ZONE_EXIT, z, lab, frame - int(rec["entry"][z])))
                    rec["entry"][z] = 0
            rec.update(inside=m, label=lab, last_seen=frame)
        for tid in sorted(self.records):
            rec = self.records[tid]
            if frame - rec["last_seen"] > p["forget_after"]:
                for z in range(Z):
                    if rec["inside"] >> z & 1:
                        events.append((tid, ZONE_FORGET, z, rec["label"], rec["last_seen"] - int(rec["entry"][z])))
                del self.records[tid]
        self.frame += 1
        return inside, occ, events

    def export(self):
        """lwdetr_zones_export's result as a dict of numpy arrays, the records in ascending id."""
        L, Z = len(self.lines), len(self.polys)
        ids = sorted(self.records)
        r = [self.records[i] for i in ids]
        return dict(frame=self.frame, overflow=self.overflow,
                    line_counts=self.line_counts[:L].astype(np.int32), entries=self.entries[:Z].astype(np.int32),
                    ids=np.array(ids, np.int32), last_seen=np.array([x["last_seen"] for x in r], np.int32),
                    labels=np.array([x["label"] for x in r], np.int32),
                    sides=np.array([x["sides"][:L] for x in r], np.int8).reshape(len(r), L),
                    inside=np.array([x["inside"] for x in r], np.uint32),
                    entry=np.array([x["entry"][:Z] for x in r], np.int32).reshape(len(r), Z))


def events_array(events, max_events):
    """A frame's events as the kernel writes them: int32 [max_events, 5], unused rows zero; and the true count."""
    out = np.zeros((max_events, 5), np.int32)
    n = min(len(events), max_events)
    if n:
        out[:n] = np.array(events[:n], np.int64).astype(np.int32)
    return out, len(events)


def regular_polygon(cx, cy, r, n, phase=0.0):
    """n vertices on a circle: a convex test zone."""
    a = phase + 2 * np.pi * np.arange(n) / n
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1)


def star(cx, cy, r_out, r_in, points, phase=0.0):
    """A concave star of 2 * points vertices."""
    a = phase + np.pi * np.arange(2 * points) / points
    r = np.where(np.arange(2 * points) % 2 == 0, r_out, r_in)
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1)


def layout(seed, size=(1080, 1920), lines=4, polygons=8, vertices=16):
    """A seeded geometry for a size[0] x size[1] frame: `lines` random segments and `polygons` polygons of `vertices`
    vertices (stars when even, so concave, else jittered circles)."""
    rng = np.random.default_rng(seed)
    H, W = size
    ln = []
    while len(ln) < lines:
        a = rng.uniform((0, 0), (W, H))
        b = rng.uniform((0, 0), (W, H))
        if np.hypot(*(b - a)) > 0.2 * W:
            ln.append((a[0], a[1], b[0], b[1]))
    ps = []
    for _ in range(polygons):
        cx, cy, r = rng.uniform(0.15 * W, 0.85 * W), rng.uniform(0.15 * H, 0.85 * H), rng.uniform(0.05, 0.3) * H
        if vertices % 2 == 0:
            ps.append(star(cx, cy, r, r * rng.uniform(0.3, 0.9), vertices // 2, rng.uniform(0, 1)))
        else:
            ps.append(regular_polygon(cx, cy, r, vertices, rng.uniform(0, 1)) + rng.normal(0, 0.05 * r, (vertices, 2)))
    return ln, ps
