"""Multi-object tracking (lwdetr_track in include/lwdetr_b200.h), restated in numpy for the tests: ByteTrack's
BYTETracker.update (non-MOT20 settings) per camera stream, with the deviations the header states.

Everything is float64 with each operation rounded on its own (numpy does not fuse), in the order the header fixes:
  Kalman filter in xyah as four independent (position, velocity) pairs with covariance (P, C, V) per coordinate;
  IoU without the +1 pixel term; costs 1 - iou (or 1 - iou * score with score fusion);
  assignment by the shortest-augmenting-path Hungarian method on the n x (m + n) matrix whose column m + i is row i's own
  "unmatched" column of cost L (solve()), which is what lap.lapjv(cost, extend_cost=True, cost_limit=L) returns up to ties.

With a camera motion (lwdetr_track_ex), warp() moves every track after the predict, in the header's operation order.

With appearance (lwdetr_track_reid, BoT-SORT's with_reid path), Stream takes reid parameters (reid_params()) and each
frame's entry embeddings: each track keeps an fp32 unit embedding, and the pool x high and unconfirmed x rest associations
take min(IoU cost, appearance cost) (appearance_cost()); fixed_sum() is the header's fixed summation order.

scene() is a seeded generator of synthetic detection sequences for the tests and the benchmark, optionally seen through a
moving camera (camera_path()).
"""
import numpy as np

TRACKED, LOST = 1, 2
WP, WV = 1.0 / 20, 1.0 / 160
INF = np.inf

DEFAULTS = dict(track_thresh=0.5, low_thresh=0.1, new_track_thresh=None, match_thresh=0.8, second_thresh=0.5,
                unconfirmed_thresh=0.7, duplicate_thresh=0.15, track_buffer=30, frame_rate=30, fuse_score=1, class_aware=0,
                capacity=512)


def params(**kw):
    """The parameter block with ByteTrack's defaults; thresholds are float32, as lwdetr_track_params holds them."""
    bad = set(kw) - set(DEFAULTS)
    if bad:
        raise TypeError("unknown tracker parameters: %s" % ", ".join(sorted(bad)))
    p = dict(DEFAULTS)
    p.update({k: v for k, v in kw.items()})
    if p["new_track_thresh"] is None:
        p["new_track_thresh"] = p["track_thresh"] + 0.1
    for k in ("track_thresh", "low_thresh", "new_track_thresh", "match_thresh", "second_thresh", "unconfirmed_thresh",
              "duplicate_thresh"):
        p[k] = np.float32(p[k])
    for k in ("track_buffer", "frame_rate", "fuse_score", "class_aware", "capacity"):
        p[k] = int(p[k])
    p["max_time_lost"] = int(p["frame_rate"] / 30.0 * p["track_buffer"])
    return p


# ---------------------------------------------------------------------------------------------- Kalman filter (xyah)
class Track:
    __slots__ = ("id", "state", "activated", "start", "end", "score", "label", "index", "p", "v", "P", "C", "V", "emb")

    def box(self):
        """xyxy float64 from the state: w = a * h, x1 = cx - w / 2, y1 = cy - h / 2, x2 = x1 + w, y2 = y1 + h."""
        cx, cy, a, h = self.p
        w = a * h
        x1 = cx - w / 2
        y1 = cy - h / 2
        return np.array([x1, y1, x1 + w, y1 + h])


def measurement(box):
    """xyah float64 of an xyxy fp32 box: w = x2 - x1, h = y2 - y1, (x1 + w / 2, y1 + h / 2, w / h, h)."""
    x1, y1, x2, y2 = (np.float64(c) for c in box)
    w = x2 - x1
    h = y2 - y1
    return np.array([x1 + w / 2, y1 + h / 2, w / h, h])


def _std(h, w, fixed):
    """(w * h, w * h, fixed, w * h)."""
    s = w * h
    return np.array([s, s, fixed, s])


def initiate(t, z):
    h = z[3]
    t.p = z.copy()
    t.v = np.zeros(4)
    sp = _std(h, 2 * WP, 1e-2)
    sv = _std(h, 10 * WV, 1e-5)
    t.P = sp * sp
    t.C = np.zeros(4)
    t.V = sv * sv


def predict(t):
    if t.state != TRACKED:
        t.v[3] = 0.0
    h = t.p[3]
    sp = _std(h, WP, 1e-2)
    sv = _std(h, WV, 1e-5)
    t.p = t.p + t.v
    t.P = ((t.P + (t.C + t.C)) + t.V) + sp * sp
    t.C = t.C + t.V
    t.V = t.V + sv * sv


def kalman_update(t, z):
    h = t.p[3]
    sr = _std(h, WP, 1e-1)
    S = t.P + sr * sr
    Kp = t.P / S
    Kv = t.C / S
    y = z - t.p
    t.p = t.p + Kp * y
    t.v = t.v + Kv * y
    t.P = t.P - (Kp * Kp) * S
    t.C = t.C - (Kp * Kv) * S
    t.V = t.V - (Kv * Kv) * S


def warp(t, m):
    """Camera motion (a, b, tx, ty) applied to a track: centre by the similarity, velocity by its linear part, h and v_h by
    s = sqrt(a^2 + b^2), (P, C, V) of x, y and h by s^2; the aspect keeps its state."""
    a, b, tx, ty = (np.float64(x) for x in m)
    s2 = a * a + b * b
    s = np.sqrt(s2)
    p, v = t.p.copy(), t.v.copy()
    cx, cy, vx, vy = p[0], p[1], v[0], v[1]
    p[0] = (a * cx - b * cy) + tx
    p[1] = (b * cx + a * cy) + ty
    v[0] = a * vx - b * vy
    v[1] = b * vx + a * vy
    p[3] = s * p[3]
    v[3] = s * v[3]
    t.p, t.v = p, v
    t.P, t.C, t.V = t.P.copy(), t.C.copy(), t.V.copy()
    for q in (0, 1, 3):
        t.P[q] = s2 * t.P[q]
        t.C[q] = s2 * t.C[q]
        t.V[q] = s2 * t.V[q]


# ---------------------------------------------------------------------------------------------- costs and assignment
def iou(a, b):
    """IoU of float64 xyxy boxes a [n, 4] x b [m, 4] -> [n, m]; 0 where either area or the union is not > 0."""
    a = np.asarray(a, np.float64).reshape(-1, 4)[:, None, :]
    b = np.asarray(b, np.float64).reshape(-1, 4)[None, :, :]
    ix = np.fmax(0.0, np.fmin(a[..., 2], b[..., 2]) - np.fmax(a[..., 0], b[..., 0]))
    iy = np.fmax(0.0, np.fmin(a[..., 3], b[..., 3]) - np.fmax(a[..., 1], b[..., 1]))
    inter = ix * iy
    aa = np.fmax(0.0, a[..., 2] - a[..., 0]) * np.fmax(0.0, a[..., 3] - a[..., 1])
    ab = np.fmax(0.0, b[..., 2] - b[..., 0]) * np.fmax(0.0, b[..., 3] - b[..., 1])
    union = (aa + ab) - inter
    ok = (aa > 0) & (ab > 0) & (union > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(ok, inter / np.where(ok, union, 1.0), 0.0)


def cost_matrix(tboxes, tlabels, dboxes, dscores, dlabels, L, fuse, class_aware, emb=None):
    """[n, m] float64: 1 - iou (fuse: 1 - iou * score), +inf where the pair is not admissible (cost >= L, or labels
    differ under class_aware).  emb: the [n, m] appearance cost emb' (appearance_cost()); the cost is then
    min(that cost, emb')."""
    n, m = len(tboxes), len(dboxes)
    if n == 0 or m == 0:
        return np.full((n, m), INF)
    io = iou(tboxes, np.asarray(dboxes, np.float64))
    c = 1.0 - io * np.asarray(dscores, np.float32).astype(np.float64)[None, :] if fuse else 1.0 - io
    if emb is not None:
        c = np.minimum(c, emb)
    ok = c < np.float64(L)
    if class_aware:
        ok &= np.asarray(tlabels)[:, None] == np.asarray(dlabels)[None, :]
    return np.where(ok, c, INF)


def solve(cost, L):
    """Shortest-augmenting-path Hungarian method (the classic potentials formulation) on the n x (m + n) matrix
    [cost | D], D[i, i] = L and +inf elsewhere; rows in order, each Dijkstra step taking the unused column with the
    smallest slack, lowest column on ties.  Returns (match [n] int: the column of each row or -1, u [n] and v [m]: the
    final row and real-column potentials)."""
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    match = np.full(n, -1, np.int64)
    if n == 0 or m == 0:
        return match, np.zeros(n), np.zeros(m)
    M = m + n
    a = np.full((n + 1, M + 1), INF)                  # 1-based, as the classic statement
    a[1:, 1:m + 1] = cost
    a[np.arange(1, n + 1), m + np.arange(1, n + 1)] = np.float64(L)
    u = np.zeros(n + 1)
    v = np.zeros(M + 1)
    p = np.zeros(M + 1, np.int64)                     # p[j]: row matched to column j, 0 = free
    way = np.zeros(M + 1, np.int64)
    for i in range(1, n + 1):
        p[0] = i
        j0 = 0
        minv = np.full(M + 1, INF)
        used = np.zeros(M + 1, bool)
        while True:
            used[j0] = True
            i0 = p[j0]
            free = ~used
            free[0] = False
            cur = (a[i0] - u[i0]) - v
            better = free & (cur < minv)
            minv[better] = cur[better]
            way[better] = j0
            cand = np.where(free, minv, INF)
            j1 = int(np.argmin(cand))                 # first minimum: lowest column on ties
            delta = cand[j1]
            ju = np.nonzero(used)[0]
            u[p[ju]] += delta                         # distinct rows
            v[ju] -= delta
            minv[free] -= delta
            j0 = j1
            if p[j0] == 0:
                break
        while True:
            j1 = way[j0]
            p[j0] = p[j1]
            j0 = j1
            if j0 == 0:
                break
    for j in range(1, m + 1):
        if p[j]:
            match[p[j] - 1] = j - 1
    return match, u[1:].copy(), v[1:m + 1].copy()


def components(cost):
    """Connected components of the admissible (finite) entries: (list of row index arrays, list of column index arrays),
    each in ascending order, one pair per component that has a row; columns without an admissible entry are left out."""
    n, m = cost.shape
    parent = list(range(n + m))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for i, j in zip(*np.nonzero(np.isfinite(cost))):
        a, b = find(int(i)), find(n + int(j))
        if a != b:
            parent[max(a, b)] = min(a, b)
    groups = {}
    for x in range(n + m):
        groups.setdefault(find(x), []).append(x)
    rows, cols = [], []
    for g in sorted(groups):
        r = [x for x in groups[g] if x < n]
        if r:
            rows.append(np.array(r, np.int64))
            cols.append(np.array([x - n for x in groups[g] if x >= n], np.int64))
    return rows, cols


def solve_by_components(cost, L):
    """solve() applied to each connected component on its own (rows and columns kept in their global order): the same
    match, u and v bits as solve() on the whole matrix, because one row's search never leaves its component."""
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    match, u, v = np.full(n, -1, np.int64), np.zeros(n), np.zeros(m)
    for r, c in zip(*components(cost)):
        if len(c) == 0:                               # a row alone takes its own column: slack L
            u[r] = np.float64(L)
            continue
        mm, uu, vv = solve(cost[np.ix_(r, c)], L)
        match[r] = np.where(mm >= 0, c[np.maximum(mm, 0)], -1)
        u[r] = uu
        v[c] = vv
    return match, u, v


# ---------------------------------------------------------------------------------------------- appearance
REID_DEFAULTS = dict(embedding_dim=256, proximity_thresh=0.5, appearance_thresh=0.25, ema_alpha=0.9)


def reid_params(**kw):
    """lwdetr_reid_params with BoT-SORT's defaults; thresholds and alpha are float32, as the struct holds them."""
    bad = set(kw) - set(REID_DEFAULTS)
    if bad:
        raise TypeError("unknown appearance parameters: %s" % ", ".join(sorted(bad)))
    r = dict(REID_DEFAULTS)
    r.update(kw)
    for k in ("proximity_thresh", "appearance_thresh", "ema_alpha"):
        r[k] = np.float32(r[k])
    r["embedding_dim"] = int(r["embedding_dim"])
    return r


def fixed_sum(x):
    """The header's summation order of D float64 terms: 32 partial sums from 0, partial j adding terms j, j + 32, ... in
    ascending order, then the xor butterfly 16, 8, 4, 2, 1 (lane j adds lane j ^ o; addition commutes, so every lane
    ends with the same bits); the value of lane 0."""
    x = np.asarray(x, np.float64)
    p = np.zeros(32)
    for j0 in range(0, len(x), 32):
        c = x[j0:j0 + 32]
        p[:len(c)] = p[:len(c)] + c
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[lane ^ o]
    return p[0]


def fixed_norm(x):
    x = np.asarray(x, np.float64)
    return np.sqrt(fixed_sum(x * x))


def fixed_dot(a, b):
    return fixed_sum(np.asarray(a, np.float64) * np.asarray(b, np.float64))


def entry_norms(emb):
    """ne of every entry [k, D] (widened exactly to float64); 0 where the entry has no appearance (ne not finite or not
    > 0)."""
    ne = np.array([fixed_norm(e) for e in np.asarray(emb, np.float64)]) if len(emb) else np.zeros(0)
    return np.where(np.isfinite(ne) & (ne > 0), ne, 0.0)


def appearance_cost(tracks, tboxes, dets, dboxes, emb, ne, r):
    """[n, m] emb': max(0, 1 - dot(t, e) / ne) / 2 where the track and the entry have appearance, (1 - iou) <=
    proximity_thresh and that value <= appearance_thresh; 1 elsewhere."""
    out = np.ones((len(tracks), len(dets)))
    if len(tracks) == 0 or len(dets) == 0:
        return out
    io = iou(tboxes, dboxes)
    prox, app = np.float64(r["proximity_thresh"]), np.float64(r["appearance_thresh"])
    for i, t in enumerate(tracks):
        if t.emb is None:
            continue
        for j, d in enumerate(dets):
            if ne[d] > 0 and 1.0 - io[i, j] <= prox:
                e = np.float64(max(0.0, 1.0 - fixed_dot(t.emb, emb[d]) / ne[d])) / 2.0
                out[i, j] = e if e <= app else 1.0
    return out


def ema(t, e, ne, r):
    """A track's embedding after an update by an entry with appearance: e / ne at first, else s = alpha t + (1 - alpha)
    e / ne normalised in the fixed order (unchanged when |s| is not finite or not > 0); fp32."""
    f = np.asarray(e, np.float64) / ne
    if t.emb is None:
        t.emb = f.astype(np.float32)
        return
    a = np.float64(r["ema_alpha"])
    s = a * t.emb.astype(np.float64) + (1.0 - a) * f
    n = fixed_norm(s)
    if np.isfinite(n) and n > 0:
        t.emb = (s / n).astype(np.float32)


# ---------------------------------------------------------------------------------------------- one stream
class Stream:
    """The tracker state of one camera stream: tracked and lost lists in ByteTrack's list order.  r: reid_params() for
    the appearance mode (lwdetr_track_reid), None for ByteTrack."""

    def __init__(self, p, r=None):
        self.p = p
        self.r = r
        self.reset()

    def reset(self):
        self.frame, self.next_id, self.overflow = 1, 1, 0
        self.tracked, self.lost = [], []
        self.dropped = dict(tracked=0, birth=0, lost=0)       # duplicate removals so far (step 8), for the tests

    def _cost(self, tracks, dets, L, fuse, e, app=None):
        scores, labels, boxes = e
        tb = np.array([t.box() for t in tracks]).reshape(-1, 4)
        db = boxes[dets].reshape(-1, 4)
        emb = None if app is None else appearance_cost(tracks, tb, dets, db.astype(np.float64), app[0], app[1], self.r)
        return cost_matrix(tb, [t.label for t in tracks], db, scores[dets], labels[dets], L, fuse, self.p["class_aware"], emb)

    def _update(self, t, d, e, app=None):
        """app: (embeddings, norms) for an update by a high entry in the appearance mode; a low entry leaves the
        track's embedding as it is."""
        scores, labels, boxes = e
        kalman_update(t, measurement(boxes[d]))
        t.state, t.activated, t.end = TRACKED, True, self.frame
        t.score, t.label, t.index = scores[d], labels[d], int(d)
        if app is not None and app[1][d] > 0:
            ema(t, app[0][d], app[1][d], self.r)

    def update(self, scores, labels, boxes, motion=None, embeddings=None):
        """One frame: scores fp32 [k], labels int32 [k], boxes fp32 [k, 4] (xyxy) -> the output tracks, a list of
        (id, score fp32, label, box fp32 [4], index).  motion: the frame's camera motion (a, b, tx, ty) or None.
        embeddings: [k, D] entry embeddings (values exactly widened to float64) in the appearance mode, None for
        none (then no entry has appearance)."""
        p, frame = self.p, self.frame
        scores = np.asarray(scores, np.float32).reshape(-1)
        labels = np.asarray(labels).astype(np.int32).reshape(-1)
        boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
        e = (scores, labels, boxes)
        app = None
        if self.r is not None:
            emb = np.zeros((len(scores), self.r["embedding_dim"])) if embeddings is None else np.asarray(embeddings, np.float64)
            ne = np.zeros(len(scores)) if embeddings is None else entry_norms(emb)
            app = (emb, ne)
        elif embeddings is not None:
            raise ValueError("embeddings given to a stream without appearance parameters")
        bd = boxes.astype(np.float64)
        with np.errstate(invalid="ignore"):
            valid = np.isfinite(bd).all(1) & (bd[:, 2] - bd[:, 0] > 0) & (bd[:, 3] - bd[:, 1] > 0)
        high = np.nonzero(valid & (scores > p["track_thresh"]))[0]
        low = np.nonzero(valid & (scores > p["low_thresh"]) & (scores < p["track_thresh"]))[0]

        unconf = [t for t in self.tracked if not t.activated]
        pool = [t for t in self.tracked if t.activated] + self.lost
        for t in pool:
            predict(t)
        if motion is not None:
            for t in self.tracked + self.lost:
                warp(t, motion)
        # 1. pool x high detections
        m1, _, _ = solve(self._cost(pool, high, p["match_thresh"], p["fuse_score"], e, app), p["match_thresh"])
        refound = []
        for t, c in zip(pool, m1):
            if c >= 0:
                if t.state == LOST:
                    refound.append(t)
                self._update(t, high[c], e, app)
        used = np.zeros(len(high), bool)
        used[m1[m1 >= 0]] = True
        rest = high[~used]
        # 2. the pool's unmatched Tracked tracks x low detections, no score fusion
        r_tracked = [t for t, c in zip(pool, m1) if c < 0 and t.state == TRACKED]
        m2, _, _ = solve(self._cost(r_tracked, low, p["second_thresh"], False, e), p["second_thresh"])
        new_lost = []
        for t, c in zip(r_tracked, m2):
            if c >= 0:
                self._update(t, low[c], e)
            else:
                t.state = LOST
                new_lost.append(t)
        # 3. unconfirmed tracks x the high detections left
        m3, _, _ = solve(self._cost(unconf, rest, p["unconfirmed_thresh"], p["fuse_score"], e, app), p["unconfirmed_thresh"])
        removed = set()
        for t, c in zip(unconf, m3):
            if c >= 0:
                self._update(t, rest[c], e, app)
            else:
                removed.add(id(t))
        used = np.zeros(len(rest), bool)
        used[m3[m3 >= 0]] = True
        rest = rest[~used]
        # 6. ageing (counted before births: capacity applies to the lists this frame leaves)
        ref = {id(t) for t in refound}
        aged = {id(t) for t in self.lost if id(t) not in ref and frame - t.end > p["max_time_lost"]}
        live = len(self.tracked) + len(self.lost) - len(removed) - len(aged)
        # 5. births
        births = []
        for d in rest:
            if scores[d] >= p["new_track_thresh"]:
                if live + len(births) >= p["capacity"]:
                    self.overflow += 1
                    continue
                t = Track()
                t.id, self.next_id = self.next_id, self.next_id + 1
                t.state, t.activated, t.start, t.end = TRACKED, frame == 1, frame, frame
                t.score, t.label, t.index = scores[d], labels[d], int(d)
                initiate(t, measurement(boxes[d]))
                t.emb = None
                if app is not None and app[1][d] > 0:
                    ema(t, app[0][d], app[1][d], self.r)
                births.append(t)
        # 7. new lists
        tracked = [t for t in self.tracked if t.state == TRACKED and id(t) not in removed] + births + refound
        lost = [t for t in self.lost if id(t) not in ref and id(t) not in aged] + new_lost
        # 8. duplicates between the two lists
        if tracked and lost:
            tb = np.array([t.box() for t in tracked])
            lb = np.array([t.box() for t in lost])
            dup = (1.0 - iou(tb, lb)) < np.float64(p["duplicate_thresh"])
            if p["class_aware"]:
                dup &= np.array([t.label for t in tracked])[:, None] == np.array([t.label for t in lost])[None, :]
            da, db = set(), set()
            for a, b in zip(*np.nonzero(dup)):
                if tracked[a].end - tracked[a].start > lost[b].end - lost[b].start:
                    db.add(b)
                else:
                    da.add(a)
            born = {id(t) for t in births}
            self.dropped["birth"] += sum(id(tracked[a]) in born for a in da)
            self.dropped["tracked"] += sum(id(tracked[a]) not in born for a in da)
            self.dropped["lost"] += len(db)
            tracked = [t for i, t in enumerate(tracked) if i not in da]
            lost = [t for i, t in enumerate(lost) if i not in db]
        self.tracked, self.lost = tracked, lost
        self.frame += 1
        return [(t.id, np.float32(t.score), int(t.label), t.box().astype(np.float32), t.index) for t in tracked if t.activated]

    def update_flow(self, measurements, motion=None):
        """One flow frame (lwdetr_track_flow): measurements[j] = (status, z) for the j-th activated track of the tracked
        list, z the float64 xyah measurement (flow_spec.measure); a track past the list given is SKIPPED.  Status 0 (OK)
        updates the track (score and label kept, index -1, end = frame); any other makes it Lost.  Unconfirmed tracks are
        carried; no births.  Returns the output tracks as update() does."""
        p, frame = self.p, self.frame
        conf = [t for t in self.tracked if t.activated]
        for t in conf + self.lost:
            predict(t)
        if motion is not None:
            for t in self.tracked + self.lost:
                warp(t, motion)
        new_lost = []
        for j, t in enumerate(conf):
            st, z = measurements[j] if j < len(measurements) else (5, None)
            if st == 0:
                kalman_update(t, np.asarray(z, np.float64))
                t.end, t.index = frame, -1
            else:
                t.state = LOST
                new_lost.append(t)
        tracked = [t for t in self.tracked if t.state == TRACKED]
        lost = [t for t in self.lost if not frame - t.end > p["max_time_lost"]] + new_lost
        if tracked and lost:
            dup = (1.0 - iou(np.array([t.box() for t in tracked]), np.array([t.box() for t in lost]))) < np.float64(p["duplicate_thresh"])
            if p["class_aware"]:
                dup &= np.array([t.label for t in tracked])[:, None] == np.array([t.label for t in lost])[None, :]
            da, db = set(), set()
            for a, b in zip(*np.nonzero(dup)):
                if tracked[a].end - tracked[a].start > lost[b].end - lost[b].start:
                    db.add(b)
                else:
                    da.add(a)
            tracked = [t for i, t in enumerate(tracked) if i not in da]
            lost = [t for i, t in enumerate(lost) if i not in db]
        self.tracked, self.lost = tracked, lost
        self.frame += 1
        return [(t.id, np.float32(t.score), int(t.label), t.box().astype(np.float32), -1) for t in tracked if t.activated]

    def export(self):
        """Every record in list order (tracked, then lost) as dicts with the float64 state."""
        return [dict(id=t.id, state=t.state, activated=int(t.activated), start=t.start, end=t.end, score=np.float32(t.score),
                     label=int(t.label), index=t.index, mean=np.concatenate([t.p, t.v]), cov=np.concatenate([t.P, t.C, t.V]))
                for t in self.tracked + self.lost]

    def export_embeddings(self):
        """The fp32 embedding of every record in list order (tracked, then lost), None for a track without one."""
        return [t.emb for t in self.tracked + self.lost]


def outputs_array(outs, max_out):
    """Output tracks of one frame as the kernel's padded arrays: (ids, scores, labels, boxes, index, count), unused slots
    id 0, score 0, label -1, zero box, index -1; count = min(len, max_out)."""
    n = min(len(outs), max_out)
    ids = np.zeros(max_out, np.int32)
    sc = np.zeros(max_out, np.float32)
    lab = np.full(max_out, -1, np.int32)
    bx = np.zeros((max_out, 4), np.float32)
    ix = np.full(max_out, -1, np.int32)
    for i, (tid, s, l, b, d) in enumerate(outs[:n]):
        ids[i], sc[i], lab[i], bx[i], ix[i] = tid, s, l, b, d
    return ids, sc, lab, bx, ix, n


# ---------------------------------------------------------------------------------------------- synthetic scenes
CAMERA = dict(seed=0, pan=10.0, shake=4.0, zoom=0.004, rotate=0.15)


def camera_path(frames, size, seed=0, pan=10.0, shake=4.0, zoom=0.004, rotate=0.15):
    """A seeded moving camera: per frame the similarity (a, b, tx, ty) from the previous frame's pixels to this one's
    (frame 0: the identity).  Pans of +-pan px per frame (one third of it vertically) that start and stop abruptly every 10
    to 40 frames and turn back before the view drifts far, hand shake of `shake` px (std of the camera's offset), a slow
    zoom with per-frame log-scale std `zoom` and a slow roll with per-frame std `rotate` degrees, both about the frame
    centre.  Returns float64 [frames, 4]."""
    rng = np.random.default_rng(seed)
    H, W = size
    cx, cy = W / 2.0, H / 2.0
    out = np.zeros((frames, 4))
    out[0] = (1.0, 0.0, 0.0, 0.0)
    off = np.zeros(2)
    vel = np.zeros(2)
    left = 0
    jit = np.zeros(2)
    ls = th = 0.0
    for f in range(1, frames):
        if left == 0:
            left = int(rng.integers(10, 41))
            choice = int(rng.integers(-1, 2))
            if abs(off[0]) > 0.15 * W:
                choice = -int(np.sign(off[0]))
            vel = np.array([choice * pan, rng.choice([-1, 0, 1]) * pan / 3])
            if abs(off[1]) > 0.15 * H:
                vel[1] = -np.sign(off[1]) * pan / 3
        left -= 1
        off = off + vel
        j = rng.normal(0, shake, 2)
        dls = 0.9 * ls + rng.normal(0, zoom) - ls
        dth = 0.9 * th + rng.normal(0, rotate) - th
        ls, th = ls + dls, th + dth
        s, t = np.exp(dls), np.deg2rad(dth)
        a, b = s * np.cos(t), s * np.sin(t)
        d = vel + j - jit
        jit = j
        out[f] = (a, b, cx - (a * cx - b * cy) + d[0], cy - (b * cx + a * cy) + d[1])
    return out


def scene(seed, frames, objects=20, k=None, ncls=3, size=(1080, 1920), clutter=3, miss=0.05, low_dip=0.1, occlusion=0.02,
          crossing=True, echo=0.0, camera=None, truth=False, crossings=1, appearance=None):
    """Seeded synthetic detections: `objects` ground-truth boxes alive at a time on average, moving at constant velocity with
    small accelerations, born and dying over the sequence; per frame each visible object gives a detection with jitter
    (score mostly high, dipping into the low band with probability low_dip), is missed with probability `miss`, and starts
    an occlusion (no detection for 1 to 80 frames, around ByteTrack's 30-frame buffer) with probability `occlusion`.  Pairs
    of objects cross each other (crossing).  `clutter` random boxes per frame on average at low to mid scores.  With
    probability `echo` per frame an object starts a spell of 2 to 11 frames in which it also gives a second detection a few
    pixels to the side (IoU about 0.9 with the first): such echoes start tracks on top of tracks, which the duplicate removal
    between the tracked and the lost list then resolves.  Returns a
    list of (scores fp32 [k_f], labels int32 [k_f], boxes fp32 [k_f, 4]) in shuffled order, or with k given, padded to k
    entries (score 0, zero box) or cut to its first k.
    camera (a dict of camera_path's options, CAMERA the defaults): the same objects and detections seen through a moving
    camera; every box is mapped by the camera's accumulated similarity (centre by the similarity, sides by its scale).  The
    camera draws from its own generator, so the scene's draws are those of the still scene.  truth: also give the object of
    each entry (int32 per entry, -1 for clutter and echoes).  With camera or truth the result is (frames, motion float64
    [frames, 4] or None, truth or None).
    crossings: the number of object pairs aimed at each other (with crossing), at heights spread over the frame.
    appearance (a dict of appearance_embeddings' options, APPEARANCE the defaults): also an embedding per entry, float32
    [k_f, dim] per frame; the result is then (frames, motion, truth, embeddings).  The embeddings
    draw from their own generator, so the scene's draws are those of the scene without them."""
    rng = np.random.default_rng(seed)
    H, W = size
    objs = []
    gid = [0]
    motion = None if camera is None else camera_path(frames, size, **camera)
    cam = np.array([1.0, 0.0, 0.0, 0.0])

    def spawn(t0):
        h = rng.uniform(30, 300)
        w = h * rng.uniform(0.3, 1.2)
        o = dict(cx=rng.uniform(w, W - w), cy=rng.uniform(h, H - h), w=w, h=h, vx=rng.normal(0, 4), vy=rng.normal(0, 2),
                 label=int(rng.integers(ncls)), die=t0 + int(rng.integers(40, 4 * frames + 40)), hidden=0, gid=gid[0])
        gid[0] += 1
        objs.append(o)
    for _ in range(objects):
        spawn(0)
    for i in range(min(crossings, objects // 2) if crossing else 0):     # pairs of objects aimed at each other
        a, b = objs[2 * i], objs[2 * i + 1]
        cy = H * 0.5 if crossings == 1 else H * (0.15 + 0.7 * i / (crossings - 1))
        a.update(cx=W * 0.3, cy=cy, vx=6.0, vy=0.0)
        b.update(cx=W * 0.7, cy=cy + 10, vx=-6.0, vy=0.0, h=a["h"] * 1.1, w=a["w"] * 0.9)
        if crossings > 1:                      # one class per pair, so that class-aware gating cannot tell them apart
            b["label"] = a["label"]
    out, gts = [], []
    for f in range(frames):
        if motion is not None:                 # accumulated camera: the previous one followed by this frame's motion
            a, b, tx, ty = motion[f]
            ca, cb, ctx, cty = cam
            cam = np.array([a * ca - b * cb, b * ca + a * cb, (a * ctx - b * cty) + tx, (b * ctx + a * cty) + ty])
        objs = [o for o in objs if o["die"] > f and -o["w"] < o["cx"] < W + o["w"] and -o["h"] < o["cy"] < H + o["h"]]
        while len(objs) < objects and rng.random() < 0.3:
            spawn(f)
        det = []
        for o in objs:
            o["vx"] += rng.normal(0, 0.3)
            o["vy"] += rng.normal(0, 0.2)
            o["cx"] += o["vx"]
            o["cy"] += o["vy"]
            if o["hidden"] > 0:
                o["hidden"] -= 1
                continue
            if rng.random() < occlusion:
                o["hidden"] = int(rng.integers(1, 80))
                continue
            if rng.random() < miss:
                continue
            j = 0.03 * o["h"]
            cx, cy = o["cx"] + rng.normal(0, j), o["cy"] + rng.normal(0, j)
            w, h = o["w"] * (1 + rng.normal(0, 0.03)), o["h"] * (1 + rng.normal(0, 0.03))
            s = rng.uniform(0.15, 0.5) if rng.random() < low_dip else rng.uniform(0.55, 0.98)
            det.append((s, o["label"], cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, o["gid"]))
            if echo > 0:
                if o.get("echo", 0) == 0 and rng.random() < echo:
                    o["echo"] = int(rng.integers(2, 12))
                if o.get("echo", 0) > 0:
                    o["echo"] -= 1
                    dx = 0.025 * w * (1 + rng.normal(0, 0.1))
                    ew, eh = w * (1 + rng.normal(0, 0.01)), h * (1 + rng.normal(0, 0.01))     # its own size: no exact IoU ties
                    det.append((rng.uniform(0.65, 0.98), o["label"], cx + dx - ew / 2, cy - eh / 2, cx + dx + ew / 2, cy + eh / 2, -1))
        for _ in range(rng.poisson(clutter)):
            h = rng.uniform(20, 200)
            w = h * rng.uniform(0.3, 1.5)
            x, y = rng.uniform(0, W - w), rng.uniform(0, H - h)
            det.append((rng.uniform(0.05, 0.65), int(rng.integers(ncls)), x, y, x + w, y + h, -1))
        rng.shuffle(det)
        a = np.array(det, np.float64).reshape(-1, 7)
        bx = a[:, 2:6]
        if motion is not None:
            ca, cb, ctx, cty = cam
            s = np.sqrt(ca * ca + cb * cb)
            mx, my = (bx[:, 0] + bx[:, 2]) / 2, (bx[:, 1] + bx[:, 3]) / 2
            hw, hh = s * (bx[:, 2] - bx[:, 0]) / 2, s * (bx[:, 3] - bx[:, 1]) / 2
            nx, ny = (ca * mx - cb * my) + ctx, (cb * mx + ca * my) + cty
            bx = np.stack([nx - hw, ny - hh, nx + hw, ny + hh], 1)
        out.append(pad(a[:, 0].astype(np.float32), a[:, 1].astype(np.int32), bx.astype(np.float32), k))
        g = a[:, 6].astype(np.int32)
        gts.append(g if k is None else np.r_[g, np.full(max(0, k - len(g)), -1, np.int32)][:k])
    if appearance is not None:
        return out, motion, (gts if truth else None), appearance_embeddings(gts, **appearance)
    if camera is None and not truth:
        return out
    return out, motion, (gts if truth else None)


APPEARANCE = dict(seed=0, dim=64, cosine=0.9, same=False)


def appearance_embeddings(truth, seed=0, dim=64, cosine=0.9, same=False):
    """Seeded embeddings for scene(): a random unit vector per object (one shared by all objects with `same`, the
    control); per entry of an object that vector turned by exactly arccos(cosine) towards a random direction; a random
    unit vector for clutter, echoes and padding (object -1).  Each row is then scaled by a factor in [0.5, 2), so that the
    normalisation matters.  truth: the object of each entry per frame.  Returns float32 [k_f, dim] per frame."""
    rng = np.random.default_rng(seed)
    base = {}

    def unit(n):
        v = rng.normal(size=(n, dim))
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    shared = unit(1)[0]
    out = []
    for g in truth:
        e = np.zeros((len(g), dim))
        for i, o in enumerate(g):
            o = int(o)
            if o < 0:
                e[i] = unit(1)[0]
                continue
            if o not in base:
                base[o] = shared if same else unit(1)[0]
            u = base[o]
            n = rng.normal(size=dim)
            n -= (n @ u) * u
            n /= np.linalg.norm(n)
            e[i] = cosine * u + np.sqrt(1.0 - cosine * cosine) * n
        e *= rng.uniform(0.5, 2.0, (len(g), 1))
        out.append(e.astype(np.float32))
    return out


def id_switches(stream_outputs, truth):
    """Identity switches over a sequence: outputs of Stream.update per frame and the true object of each entry; a switch is
    an object whose matched track id differs from the id it last had."""
    last, n = {}, 0
    for outs, g in zip(stream_outputs, truth):
        for tid, _, _, _, idx in outs:
            o = int(g[idx])
            if o < 0:
                continue
            if o in last and last[o] != tid:
                n += 1
            last[o] = tid
    return n


def pad(scores, labels, boxes, k):
    """One frame's entries padded with (score 0, label 0, zero box) or cut to k entries (k None: unchanged)."""
    if k is None:
        return scores, labels, boxes
    n = min(len(scores), k)
    s = np.zeros(k, np.float32)
    lab = np.zeros(k, np.int32)
    b = np.zeros((k, 4), np.float32)
    s[:n], lab[:n], b[:n] = scores[:n], labels[:n], boxes[:n]
    return s, lab, b
