"""CPU tests of tracking by appearance (lwdetr_track_reid in include/lwdetr_b200.h, tools/track_spec.py with
reid_params()): against an independent BoT-SORT-style restatement written here from the published algorithm (scipy's
cosine cdist, np.minimum and the masks of BoTSORT.update, lapjv's extended matrix), the fixed summation order, and the
effect on identity switches in crossing scenes."""
import os
import sys

import numpy as np
import pytest
from scipy.spatial.distance import cdist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402
from test_track_cpu import KF, RefTrack, lapjv_like, ref_iou  # noqa: E402


# ------------------------------------------------------------------------------------------ the independent restatement
class RefBoTSORT:
    """BoTSORT.update with with_reid (no camera motion), list by list, with this project's stated deviations: the
    smoothed feature is kept in fp32 and the tracks and lists follow ByteTrack's as in test_track_cpu.RefByteTrack."""

    def __init__(self, p, r):
        self.p, self.r, self.frame, self.next_id = p, r, 0, 1
        self.tracked, self.lost = [], []

    def update_features(self, t, feat):
        feat = feat / np.linalg.norm(feat)
        if getattr(t, "smooth", None) is None:
            t.smooth = feat.astype(np.float32)
        else:
            a = float(self.r["ema_alpha"])
            s = a * t.smooth.astype(np.float64) + (1 - a) * feat
            t.smooth = (s / np.linalg.norm(s)).astype(np.float32)

    def dists(self, tracks, dets, fuse, reid):
        n, m = len(tracks), len(dets)
        if n == 0 or m == 0:
            return np.zeros((n, m))
        io = np.array([[ref_iou(t.tlbr(), d[2]) for d in dets] for t in tracks])
        ious_dists = 1 - io
        ious_dists_mask = ious_dists > self.r["proximity_thresh"]
        dists = 1 - io * np.array([float(d[0]) for d in dets])[None] if fuse else ious_dists.copy()
        if reid:
            emb_dists = np.ones((n, m))
            tf = [i for i, t in enumerate(tracks) if getattr(t, "smooth", None) is not None]
            df = [j for j, d in enumerate(dets) if d[4] is not None]
            if tf and df:
                c = np.maximum(0.0, cdist(np.array([tracks[i].smooth for i in tf], np.float64), np.array([dets[j][4] for j in df]), "cosine"))
                emb_dists[np.ix_(tf, df)] = c / 2.0
            emb_dists[emb_dists > self.r["appearance_thresh"]] = 1.0
            emb_dists[ious_dists_mask] = 1.0
            dists = np.minimum(dists, emb_dists)
        if self.p["class_aware"]:
            dists[np.array([t.label for t in tracks])[:, None] != np.array([d[1] for d in dets])[None]] = 1e9
        return dists

    def step(self, scores, labels, boxes, emb):
        p = self.p
        self.frame += 1
        f = self.frame
        dets = [(s, int(lab), b.astype(np.float64), i, e.astype(np.float64)) for i, (s, lab, b, e) in enumerate(zip(scores, labels, boxes, emb))
                if np.isfinite(b).all() and b[2] > b[0] and b[3] > b[1]]
        high = [d for d in dets if d[0] > p["track_thresh"]]
        low = [(*d[:4], None) for d in dets if p["low_thresh"] < d[0] < p["track_thresh"]]    # no features in round two
        z_of = lambda b: np.array([(b[0] + b[2]) / 2, (b[1] + b[3]) / 2, (b[2] - b[0]) / (b[3] - b[1]), b[3] - b[1]])

        def upd(t, d):
            t.mean, t.cov = KF.update(t.mean, t.cov, z_of(d[2]))
            t.state, t.activated, t.end, t.score, t.label, t.index = ts.TRACKED, True, f, d[0], d[1], d[3]
            if d[4] is not None:
                self.update_features(t, d[4])
        unconf = [t for t in self.tracked if not t.activated]
        pool = [t for t in self.tracked if t.activated] + self.lost
        for t in pool:
            if t.state != ts.TRACKED:
                t.mean[7] = 0
            t.mean, t.cov = KF.predict(t.mean, t.cov)
        m = lapjv_like(self.dists(pool, high, p["fuse_score"], True), float(p["match_thresh"]))
        refound = []
        for i, j in m:
            if pool[i].state == ts.LOST:
                refound.append(pool[i])
            upd(pool[i], high[j])
        mi, mj = {i for i, _ in m}, {j for _, j in m}
        high = [d for j, d in enumerate(high) if j not in mj]
        rt = [t for i, t in enumerate(pool) if i not in mi and t.state == ts.TRACKED]
        m = lapjv_like(self.dists(rt, low, False, False), float(p["second_thresh"]))
        for i, j in m:
            upd(rt[i], low[j])
        mi = {i for i, _ in m}
        new_lost = [t for i, t in enumerate(rt) if i not in mi]
        for t in new_lost:
            t.state = ts.LOST
        m = lapjv_like(self.dists(unconf, high, p["fuse_score"], True), float(p["unconfirmed_thresh"]))
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
            t = RefTrack(z_of(d[2]), d[0], d[1], d[3], f, self.next_id)
            self.update_features(t, d[4])
            births.append(t)
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


def _scene(seed, same=False, frames=300, **kw):
    kw = dict(dict(objects=40, crossings=20), **kw)
    return ts.scene(seed, frames, truth=True, appearance=dict(seed=seed, dim=64, cosine=0.9, same=same), **kw)


@pytest.mark.parametrize("seed, kw, reid", [(0, {}, {}), (1, dict(class_aware=1), {}), (2, {}, dict(appearance_thresh=0.4, ema_alpha=0.7)),
                                            (3, dict(match_thresh=0.6), dict(proximity_thresh=0.7))])
def test_spec_equals_independent_botsort_on_crossing_scenes(seed, kw, reid):
    p, r = ts.params(**kw), ts.reid_params(embedding_dim=64, **reid)
    spec, ref = ts.Stream(p, r), RefBoTSORT(p, r)
    frames, _, _, embs = _scene(seed, frames=200, objects=16, crossings=8, echo=0.03)
    n_out = 0
    for f, e in zip(frames, embs):
        a, b = spec.update(*f, embeddings=e), ref.step(*f, e)
        assert [(x[0], x[2], x[4]) for x in a] == [(x[0], x[2], x[4]) for x in b], "frame %d" % spec.frame
        for x, y in zip(a, b):
            np.testing.assert_allclose(x[3], y[3].astype(np.float32), rtol=2 ** -22)
        assert [t.id for t in spec.tracked + spec.lost] == [t.id for t in ref.tracked + ref.lost]
        for t, rt in zip(spec.tracked + spec.lost, ref.tracked + ref.lost):
            np.testing.assert_allclose(t.emb, rt.smooth, rtol=0, atol=1e-6)
        n_out += len(a)
    assert n_out > 1000


def test_without_embeddings_the_appearance_mode_is_bytetrack():
    frames, _, _, embs = _scene(5, frames=150, objects=16, crossings=8)
    a, b = ts.Stream(ts.params(), ts.reid_params(embedding_dim=64)), ts.Stream(ts.params())
    for i, f in enumerate(frames):
        e = None if i % 2 else np.zeros((len(f[0]), 64), np.float32)      # no embeddings, or only rows without appearance
        assert [(x[0], x[4]) for x in a.update(*f, embeddings=e)] == [(x[0], x[4]) for x in b.update(*f)]
    assert all(t.emb is None for t in a.tracked + a.lost)


def test_fixed_order_helpers():
    rng = np.random.default_rng(0)
    for D in (1, 31, 32, 33, 100, 256, 2048):
        x = rng.normal(size=D)
        p = np.zeros(32)
        for j in range(32):
            for i in range(j, D, 32):
                p[j] = p[j] + x[i]
        for o in (16, 8, 4, 2, 1):               # the tree lane 0 sees, written out
            p = np.array([p[j] + p[j ^ o] for j in range(32)])
        assert ts.fixed_sum(x).view(np.int64) == p[0].view(np.int64)
        y = rng.normal(size=D)
        np.testing.assert_allclose(ts.fixed_dot(x, y), np.dot(x, y), rtol=1e-14 * max(1.0, np.abs(x * y).sum() / abs(np.dot(x, y))))
        np.testing.assert_allclose(ts.fixed_norm(x), np.linalg.norm(x), rtol=1e-15 * 4)
    assert list(ts.entry_norms(np.array([[0.0, 0.0], [np.nan, 1.0], [np.inf, 0.0], [3.0, 4.0]]))) == [0.0, 0.0, 0.0, 5.0]


def test_appearance_cuts_identity_switches_in_crossing_scenes():
    """Crossing-rich scenes (20 pairs of same-class objects aimed at each other), distinct appearances: fewer identity
    switches than IoU alone for every seed.  The control, where every object looks the same, is run and printed only."""
    rows = []
    for seed in (0, 1, 2):
        got = {}
        for mode in ("iou", "reid", "same"):
            frames, _, truth, embs = _scene(seed, same=mode == "same")
            st = ts.Stream(ts.params(), None if mode == "iou" else ts.reid_params(embedding_dim=64))
            outs = [st.update(*f, embeddings=None if mode == "iou" else e) for f, e in zip(frames, embs)]
            got[mode] = ts.id_switches(outs, truth)
        rows.append(got)
        print("seed %d: identity switches IoU only %d, appearance %d, one shared appearance %d" % (seed, got["iou"], got["reid"], got["same"]))
    assert all(g["reid"] < g["iou"] for g in rows), rows
