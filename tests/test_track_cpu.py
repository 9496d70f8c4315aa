"""CPU tests of the tracker specification (tools/track_spec.py, lwdetr_track in include/lwdetr_b200.h): against an
independent list-based ByteTrack written here with an 8x8 matrix Kalman filter and scipy's assignment on lapjv's extended
matrix, the closed-form Kalman steps against the matrix form, the Hungarian method against scipy's optimum, the
per-component decomposition the kernel relies on, and the lifecycle edge cases."""
import os
import sys

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402


# ------------------------------------------------------------------------------------------ the independent restatement
class MatrixKalman:
    """ByteTrack's KalmanFilter (xyah, 8-dimensional state) in matrix form."""

    def __init__(self):
        self.F = np.eye(8)
        for i in range(4):
            self.F[i, 4 + i] = 1.0
        self.H = np.eye(4, 8)

    def initiate(self, z):
        h = z[3]
        std = [2 * ts.WP * h, 2 * ts.WP * h, 1e-2, 2 * ts.WP * h, 10 * ts.WV * h, 10 * ts.WV * h, 1e-5, 10 * ts.WV * h]
        return np.r_[z, np.zeros(4)], np.diag(np.square(std))

    def predict(self, mean, cov):
        h = mean[3]
        std = [ts.WP * h, ts.WP * h, 1e-2, ts.WP * h, ts.WV * h, ts.WV * h, 1e-5, ts.WV * h]
        return self.F @ mean, self.F @ cov @ self.F.T + np.diag(np.square(std))

    def update(self, mean, cov, z):
        h = mean[3]
        R = np.diag(np.square([ts.WP * h, ts.WP * h, 1e-1, ts.WP * h]))
        S = self.H @ cov @ self.H.T + R
        K = np.linalg.solve(S, (cov @ self.H.T).T).T
        return mean + K @ (z - self.H @ mean), cov - K @ S @ K.T


KF = MatrixKalman()


class RefTrack:
    def __init__(self, z, score, label, index, frame, tid):
        self.mean, self.cov = KF.initiate(z)
        self.score, self.label, self.index = score, label, index
        self.id, self.state, self.activated = tid, ts.TRACKED, frame == 1
        self.start = self.end = frame

    def tlbr(self):
        cx, cy, a, h = self.mean[:4]
        w = a * h
        return np.array([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2])


def ref_iou(a, b):
    x1, y1 = max(a[0], b[0]), max(a[1], b[1])
    x2, y2 = min(a[2], b[2]), min(a[3], b[3])
    inter = max(0.0, x2 - x1) * max(0.0, y2 - y1)
    aa = (a[2] - a[0]) * (a[3] - a[1])
    ab = (b[2] - b[0]) * (b[3] - b[1])
    return inter / (aa + ab - inter) if aa > 0 and ab > 0 else 0.0


def lapjv_like(cost, L):
    """lap.lapjv(cost, extend_cost=True, cost_limit=L) restated with scipy: the (n + m) square matrix with L / 2 in the
    off-diagonal blocks and 0 in the bottom-right one."""
    n, m = cost.shape
    if n == 0 or m == 0:
        return []
    ext = np.full((n + m, n + m), L / 2)
    ext[n:, m:] = 0.0
    ext[:n, :m] = np.minimum(cost, 1e6)
    r, c = linear_sum_assignment(ext)
    return [(i, j) for i, j in zip(r, c) if i < n and j < m and cost[i, j] < L]


class RefByteTrack:
    """BYTETracker.update written list by list as in ByteTrack (with this project's stated deviations)."""

    def __init__(self, p):
        self.p, self.frame, self.next_id = p, 0, 1
        self.tracked, self.lost = [], []

    def dists(self, tracks, dets, fuse):
        c = np.full((len(tracks), len(dets)), 1e9)
        for i, t in enumerate(tracks):
            for j, (s, lab, box, _) in enumerate(dets):
                if self.p["class_aware"] and t.label != lab:
                    continue
                io = ref_iou(t.tlbr(), box)
                c[i, j] = 1 - io * float(s) if fuse else 1 - io
        return c

    def step(self, scores, labels, boxes):
        p = self.p
        self.frame += 1
        f = self.frame
        dets = [(s, int(lab), b.astype(np.float64), i) for i, (s, lab, b) in enumerate(zip(scores, labels, boxes))
                if np.isfinite(b).all() and b[2] > b[0] and b[3] > b[1]]
        high = [d for d in dets if d[0] > p["track_thresh"]]
        low = [d for d in dets if p["low_thresh"] < d[0] < p["track_thresh"]]
        z_of = lambda b: np.array([(b[0] + b[2]) / 2, (b[1] + b[3]) / 2, (b[2] - b[0]) / (b[3] - b[1]), b[3] - b[1]])

        def upd(t, d):
            t.mean, t.cov = KF.update(t.mean, t.cov, z_of(d[2]))
            t.state, t.activated, t.end, t.score, t.label, t.index = ts.TRACKED, True, f, d[0], d[1], d[3]
        unconf = [t for t in self.tracked if not t.activated]
        pool = [t for t in self.tracked if t.activated] + self.lost
        for t in pool:
            if t.state != ts.TRACKED:
                t.mean[7] = 0
            t.mean, t.cov = KF.predict(t.mean, t.cov)
        m = lapjv_like(self.dists(pool, high, p["fuse_score"]), float(p["match_thresh"]))
        refound = []
        for i, j in m:
            if pool[i].state == ts.LOST:
                refound.append(pool[i])
            upd(pool[i], high[j])
        mi, mj = {i for i, _ in m}, {j for _, j in m}
        high = [d for j, d in enumerate(high) if j not in mj]
        rt = [t for i, t in enumerate(pool) if i not in mi and t.state == ts.TRACKED]
        m = lapjv_like(self.dists(rt, low, False), float(p["second_thresh"]))
        for i, j in m:
            upd(rt[i], low[j])
        mi = {i for i, _ in m}
        new_lost = [t for i, t in enumerate(rt) if i not in mi]
        for t in new_lost:
            t.state = ts.LOST
        m = lapjv_like(self.dists(unconf, high, p["fuse_score"]), float(p["unconfirmed_thresh"]))
        for i, j in m:
            upd(unconf[i], high[j])
        mi, mj = {i for i, _ in m}, {j for _, j in m}
        removed = [t for i, t in enumerate(unconf) if i not in mi]
        aged = [t for t in self.lost if t not in refound and f - t.end > p["max_time_lost"]]
        live = len(self.tracked) + len(self.lost) - len(removed) - len(aged)
        births = []
        for j, d in enumerate(high):
            if j in mj or d[0] < p["new_track_thresh"] or live + len(births) >= p["capacity"]:
                continue
            births.append(RefTrack(z_of(d[2]), d[0], d[1], d[3], f, self.next_id))
            self.next_id += 1
        tracked = [t for t in self.tracked if t.state == ts.TRACKED and t not in removed] + births + refound
        lost = [t for t in self.lost if t not in refound and t not in aged] + new_lost
        da, db = set(), set()
        for a, ta in enumerate(tracked):
            for b, tb in enumerate(lost):
                if p["class_aware"] and ta.label != tb.label:
                    continue
                if 1 - ref_iou(ta.tlbr(), tb.tlbr()) < p["duplicate_thresh"]:
                    (db.add(b) if ta.end - ta.start > tb.end - tb.start else da.add(a))
        self.tracked = [t for i, t in enumerate(tracked) if i not in da]
        self.lost = [t for i, t in enumerate(lost) if i not in db]
        return [(t.id, t.score, t.label, t.tlbr(), t.index) for t in self.tracked if t.activated]


# (seed, echo, parameters): the echo scenes start tracks on top of tracks, so step 8 (duplicates) drops tracked and lost
# tracks, and at a low match_thresh also births
SCENES = [(0, 0.0, {}), (1, 0.0, {}), (2, 0.0, dict(class_aware=1)), (3, 0.08, {}), (4, 0.08, dict(match_thresh=0.15))]


@pytest.mark.parametrize("seed, echo, kw", SCENES)
def test_spec_equals_independent_bytetrack_on_synthetic_scenes(seed, echo, kw):
    p = ts.params(**kw)
    spec, ref = ts.Stream(p), RefByteTrack(p)
    n_out, ids = 0, set()
    for f in ts.scene(seed, 320, objects=12, occlusion=0.03, echo=echo):
        a, b = spec.update(*f), ref.step(*f)
        assert [(x[0], x[2], x[4]) for x in a] == [(x[0], x[2], x[4]) for x in b], "frame %d" % spec.frame
        for x, y in zip(a, b):
            assert x[1] == np.float32(y[1])
            np.testing.assert_allclose(x[3], y[3].astype(np.float32), rtol=2 ** -22)       # output: fp32 rounding only
        assert [t.id for t in spec.tracked + spec.lost] == [t.id for t in ref.tracked + ref.lost]
        for t, r in zip(spec.tracked + spec.lost, ref.tracked + ref.lost):               # float64 state of both lists
            np.testing.assert_allclose(t.box(), r.tlbr(), rtol=1e-9)
        n_out += len(a)
        ids |= {x[0] for x in a}
    # the scenes exercise births, losses and re-finds (at match_thresh 0.15 fewer tracks stay matched)
    assert n_out > (500 if "match_thresh" in kw else 1000) and len(ids) > 15
    if echo:
        d = spec.dropped
        assert d["tracked"] >= 5 and d["lost"] >= 5, d
        assert d["birth"] >= 5 if kw else d["birth"] == 0, d


def test_scene_generator_is_seeded_and_varied():
    a, b = ts.scene(5, 50), ts.scene(5, 50)
    assert all(np.array_equal(x[2], y[2]) for x, y in zip(a, b))
    s = np.concatenate([x[0] for x in a])
    assert ((s > 0.1) & (s < 0.5)).any() and (s > 0.6).any()
    assert len(ts.scene(5, 10, k=64)[0][0]) == 64


# ------------------------------------------------------------------------------------------ Kalman
def _matrix_state(t):
    cov = np.zeros((8, 8))
    for q in range(4):
        cov[q, q], cov[q, 4 + q], cov[4 + q, q], cov[4 + q, 4 + q] = t.P[q], t.C[q], t.C[q], t.V[q]
    return np.r_[t.p, t.v], cov


def _check_state(t, mean, cov, prior):
    np.testing.assert_allclose(np.r_[t.p, t.v], mean, rtol=1e-12, atol=1e-12 * np.abs(mean).max())
    off = cov.copy()
    for q in range(4):
        blk = np.array([t.P[q], t.C[q], t.V[q]])
        want = np.array([cov[q, q], cov[q, 4 + q], cov[4 + q, 4 + q]])
        # relative to the block the step started from: the update subtracts a term of that size
        np.testing.assert_allclose(blk, want, rtol=1e-12, atol=1e-12 * max(prior[q, q], prior[4 + q, 4 + q]))
        off[q, q] = off[q, 4 + q] = off[4 + q, q] = off[4 + q, 4 + q] = 0
    assert np.abs(off).max() == 0                       # the four 2x2 blocks stay independent


def test_closed_form_kalman_equals_matrix_form_over_long_sequences():
    """Every predict and update of 5 sequences of 400 frames (10 % of them lost: v_h zeroed, no update), each step
    taken by both forms from the same state."""
    rng = np.random.default_rng(3)
    for trial in range(5):
        z = np.array([500.0, 300.0, 0.5, 120.0]) + rng.normal(0, 5, 4) * [1, 1, 0.01, 1]
        t = ts.Track()
        ts.initiate(t, z)
        mean, cov = KF.initiate(z)
        _check_state(t, mean, cov, cov)
        for step in range(400):
            lost = rng.random() < 0.1
            t.state = ts.LOST if lost else ts.TRACKED
            mean, cov = _matrix_state(t)
            if lost:
                mean[7] = 0
            ts.predict(t)
            mean, cov = KF.predict(mean, cov)
            _check_state(t, mean, cov, cov)
            if not lost:
                z = mean[:4] + rng.normal(0, 2, 4) * [1, 1, 0.005, 1]
                mean, prior = _matrix_state(t)
                ts.kalman_update(t, z)
                mean, cov = KF.update(mean, prior, z)
                _check_state(t, mean, cov, prior)


# ------------------------------------------------------------------------------------------ assignment
def _random_cost(rng, n, m, density, L, ties=False):
    c = rng.random((n, m)) * L * 1.2
    if ties:
        c = np.round(c * 8) / 8                           # many exactly equal costs
    c[rng.random((n, m)) > density] = np.inf
    c[c >= L] = np.inf
    return c


def _objective(cost, match, L):
    return sum(L - cost[i, j] for i, j in enumerate(match) if j >= 0)


@pytest.mark.parametrize("ties", [False, True])
def test_hungarian_reaches_scipy_optimum(ties):
    rng = np.random.default_rng(7 + ties)
    unique = 0
    for trial in range(150):
        n, m = int(rng.integers(1, 25)), int(rng.integers(1, 25))
        L = float(np.float32(rng.choice([0.5, 0.7, 0.8])))
        c = _random_cost(rng, n, m, rng.choice([0.1, 0.3, 1.0]), L, ties)
        match, _, _ = ts.solve(c, L)
        assert len(set(match[match >= 0])) == (match >= 0).sum()
        assert all(np.isfinite(c[i, j]) for i, j in enumerate(match) if j >= 0)
        w = np.where(np.isfinite(c), L - c, 0.0)
        r, k = linear_sum_assignment(w, maximize=True)
        best = sum(w[i, j] for i, j in zip(r, k))
        assert abs(_objective(c, match, L) - best) <= 1e-12 * max(1.0, best)
        if not ties:                                     # continuous costs: the optimum is unique
            want = np.full(n, -1)
            for i, j in zip(r, k):
                if w[i, j] > 0:
                    want[i] = j
            assert np.array_equal(match, want)
            unique += 1
    assert ties or unique == 150


def test_solving_per_component_gives_the_same_bits():
    rng = np.random.default_rng(11)
    comps = 0
    for trial in range(60):
        n, m = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        L = float(np.float32(0.8))
        c = _random_cost(rng, n, m, rng.choice([0.03, 0.08, 0.3]), L, ties=trial % 2 == 0)
        a, b = ts.solve(c, L), ts.solve_by_components(c, L)
        for x, y in zip(a, b):
            assert np.array_equal(np.asarray(x).view(np.int64), np.asarray(y).view(np.int64))
        comps += len(ts.components(c)[0])
    assert comps > 300


def test_hungarian_ties_go_to_the_lowest_column():
    L = 0.8
    c = np.full((2, 3), 0.5)
    assert list(ts.solve(c, L)[0]) == [0, 1]
    c = np.array([[0.2, 0.2], [np.inf, np.inf]])
    assert list(ts.solve(c, L)[0]) == [0, -1]


# ------------------------------------------------------------------------------------------ lifecycle
def _box(cx, cy, w=40.0, h=80.0):
    return [cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2]


def _frame(dets):
    """[(score, label, box)] -> arrays."""
    if not dets:
        return np.zeros(0, np.float32), np.zeros(0, np.int32), np.zeros((0, 4), np.float32)
    return (np.array([d[0] for d in dets], np.float32), np.array([d[1] for d in dets], np.int32),
            np.array([d[2] for d in dets], np.float32))


def test_frame_one_activation_and_confirmation_later():
    s = ts.Stream(ts.params())
    out = s.update(*_frame([(0.9, 0, _box(100, 100))]))
    assert [o[0] for o in out] == [1]                   # frame 1: activated at once
    out = s.update(*_frame([(0.9, 0, _box(101, 100)), (0.9, 0, _box(400, 100))]))
    assert [o[0] for o in out] == [1]                   # the frame-2 birth is unconfirmed
    out = s.update(*_frame([(0.9, 0, _box(102, 100)), (0.9, 0, _box(401, 100))]))
    assert sorted(o[0] for o in out) == [1, 2]


def test_unconfirmed_track_is_removed_when_unmatched():
    s = ts.Stream(ts.params())
    s.update(*_frame([(0.9, 0, _box(100, 100))]))
    s.update(*_frame([(0.9, 0, _box(100, 100)), (0.9, 0, _box(500, 100))]))
    assert len(s.tracked) == 2 and not s.tracked[1].activated
    s.update(*_frame([(0.9, 0, _box(100, 100))]))
    assert [t.id for t in s.tracked] == [1] and s.lost == []
    out = s.update(*_frame([(0.9, 0, _box(100, 100)), (0.9, 0, _box(500, 100))]))
    assert s.tracked[1].id == 3                          # a fresh id: the removed one is gone


@pytest.mark.parametrize("extra", [0, 1])
def test_lost_for_exactly_max_time_lost_is_refound_one_more_frame_removes_it(extra):
    p = ts.params(track_buffer=5)
    assert p["max_time_lost"] == 5
    s = ts.Stream(p)
    for f in range(3):
        s.update(*_frame([(0.9, 0, _box(100, 100))]))
    for f in range(5 + extra):
        s.update(*_frame([]))
    assert len(s.lost) == 1 - extra
    out = s.update(*_frame([(0.9, 0, _box(100, 100))]))
    if extra:
        assert out == [] and s.tracked[0].id == 2        # a new, unconfirmed track
    else:
        assert [o[0] for o in out] == [1] and s.tracked[0].start == 1


A, B = _box(100, 100), _box(102, 100)                      # IoU 0.905: IoU distance 0.095 < duplicate_thresh 0.15


def _lists(frames, **kw):
    """Runs the frames through the specification and the independent restatement; both must end with the same lists.
    Returns (tracked ids, lost ids, spec stream)."""
    p = ts.params(**kw)
    spec, ref = ts.Stream(p), RefByteTrack(p)
    for f in frames:
        spec.update(*_frame(f))
        ref.step(*_frame(f))
    got = ([t.id for t in spec.tracked], [t.id for t in spec.lost])
    assert got == ([t.id for t in ref.tracked], [t.id for t in ref.lost])
    return got[0], got[1], spec


# Step 8 (duplicates), case by case: (frames, parameters, (tracked ids, lost ids), drops by kind) at the end
DUPLICATE_CASES = {
    # 1 and 2 start together on A and B; only A is seen next: 2 goes lost with age 0 on top of 1 (age 1) and is dropped
    "younger_lost": ([[(0.9, 0, A), (0.9, 0, B)], [(0.9, 0, A)]], {}, ([1], []), dict(tracked=0, birth=0, lost=1)),
    # 1 starts on A at frame 1, 2 on B at frame 3 (confirmed at 4); at frame 5 only B is seen: 1 (age 3) goes lost under
    # 2 (age 2), and the younger tracked track 2 is dropped
    "younger_tracked": ([[(0.9, 0, A)], [(0.9, 0, A)], [(0.9, 0, A), (0.9, 0, B)], [(0.9, 0, A), (0.9, 0, B)], [(0.9, 0, B)]], {},
                        ([], [1]), dict(tracked=1, birth=0, lost=0)),
    # as above with 2 born at frame 2: at frame 4 both ages are 2, and the tie drops the tracked track
    "tie": ([[(0.9, 0, A)], [(0.9, 0, A), (0.9, 0, B)], [(0.9, 0, A), (0.9, 0, B)], [(0.9, 0, B)]], {}, ([], [1]),
            dict(tracked=1, birth=0, lost=0)),
    # 2 born with 1, both seen twice, then only B: lost 1 (age 2) is younger than tracked 2 (age 3) and is dropped
    "older_tracked": ([[(0.9, 0, A), (0.9, 0, B)]] * 3 + [[(0.9, 0, B)]], {}, ([2], []), dict(tracked=0, birth=0, lost=1)),
    # at match_thresh 0.1 a detection on B does not re-find the lost 1 (cost 1 - 0.905 * 0.99 > 0.1), so it starts track 2,
    # which lies on 1 and is dropped at once; its id stays used
    "birth": ([[(0.99, 0, A)]] * 5 + [[]] + [[(0.99, 0, B)]], dict(match_thresh=0.1), ([], [1]), dict(tracked=0, birth=1, lost=0)),
}


@pytest.mark.parametrize("case", sorted(DUPLICATE_CASES))
def test_duplicate_removal_keeps_the_older_track(case):
    frames, kw, survivors, dropped = DUPLICATE_CASES[case]
    tracked, lost, s = _lists(frames, **kw)
    assert (tracked, lost) == survivors and s.dropped == dropped
    if case == "birth":
        assert s.next_id == 3
    if case == "younger_tracked":
        assert s.lost[0].start == 1 and s.lost[0].end == 4


def test_class_aware_gating():
    for aware in (0, 1):
        s = ts.Stream(ts.params(class_aware=aware))
        s.update(*_frame([(0.9, 0, _box(100, 100))]))
        out = s.update(*_frame([(0.9, 1, _box(102, 100))]))
        if aware:
            assert out == [] and [t.id for t in s.lost] == [1]
        else:
            assert [(o[0], o[2]) for o in out] == [(1, 1)]


def test_degenerate_entries_are_ignored():
    s = ts.Stream(ts.params())
    bad = [[10, 10, 10, 50], [10, 10, 50, 5], [np.nan, 0, 10, 10], [0, 0, np.inf, 10]]
    out = s.update(*_frame([(0.9, 0, b) for b in bad] + [(0.9, 0, _box(100, 100))]))
    assert [(o[0], o[4]) for o in out] == [(1, 4)]


def test_refused_birth_at_capacity_takes_no_id():
    s = ts.Stream(ts.params(capacity=2))
    out = s.update(*_frame([(0.9, 0, _box(100 + 100 * i, 100)) for i in range(4)]))
    assert [o[0] for o in out] == [1, 2] and s.overflow == 2 and s.next_id == 3
    out = s.update(*_frame([(0.9, 0, _box(100, 100)), (0.9, 0, _box(200, 100)), (0.9, 0, _box(900, 100))]))
    assert s.overflow == 3 and s.next_id == 3
    s.update(*_frame([(0.9, 0, _box(100, 100))]))        # track 2 lost: still counted against the capacity
    s.update(*_frame([(0.9, 0, _box(100, 100)), (0.9, 0, _box(900, 900))]))
    assert s.overflow == 4 and s.next_id == 3
