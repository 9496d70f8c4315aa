"""GPU tests of multi-object tracking: the tracker kernel (csrc/track.cu, lwdetr_track) bit for bit against its
specification (tools/track_spec.py), outputs every frame and the float64 list state at the end; lwdetr_query_best against
lwdetr_postprocess; CUDA-graph replay; LWDETR.track against the same steps composed by hand."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import copy  # noqa: E402

import track_spec as ts  # noqa: E402
import yuv_spec  # noqa: E402
from test_track_cpu import DUPLICATE_CASES, _frame  # noqa: E402


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.view(np.int64) if a.dtype == np.float64 else a


class Pair:
    """A device tracker and one specification stream per stream id, driven together."""

    def __init__(self, num_streams, **params):
        from b200 import capi
        self.dev = capi.Tracker(num_streams, **params)
        self.spec = [ts.Stream(ts.params(**params)) for _ in range(num_streams)]
        self.outputs = 0

    def reset(self, streams):
        self.dev.reset(streams)
        for s in streams:
            self.spec[s].reset()

    def step(self, frames, streams, max_out):
        """frames: per stream id in `streams`, (scores, labels, boxes) of one common k."""
        sc = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
        lb = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
        bx = torch.from_numpy(np.stack([f[2] for f in frames])).cuda()
        got = [g.cpu().numpy() for g in self.dev.update(sc, lb, bx, streams, max_out)]
        for r, (s, f) in enumerate(zip(streams, frames)):
            want = ts.outputs_array(self.spec[s].update(*f), max_out)
            for name, g, w in zip(("ids", "scores", "labels", "boxes", "index", "count"), got, want):
                assert np.array_equal(_bits(g[r]), _bits(np.asarray(w))), "stream %d frame %d: %s" % (s, self.spec[s].frame - 1, name)
            self.outputs += want[5]

    def check_state(self):
        for s, spec in enumerate(self.spec):
            recs, fno = self.dev.export(s)
            assert fno == (spec.frame, spec.next_id, spec.overflow), s
            want = spec.export()
            assert len(recs) == len(want), s
            for g, w in zip(recs, want):
                for key in ("id", "state", "activated", "start", "end", "label", "index"):
                    assert g[key] == w[key], (s, key)
                assert _bits(np.float32(g["score"])) == _bits(np.float32(w["score"]))
                assert np.array_equal(_bits(g["mean"]), _bits(w["mean"])) and np.array_equal(_bits(g["cov"]), _bits(w["cov"])), s


def _all_low(k, rng):
    s = rng.uniform(0.11, 0.49, k).astype(np.float32)
    b = np.sort(rng.uniform(0, 1000, (k, 4)).astype(np.float32).reshape(k, 2, 2), axis=1).transpose(0, 2, 1).reshape(k, 4)
    return s, np.zeros(k, np.int32), b


def test_64_streams_over_220_frames_with_absent_streams_resets_and_special_frames():
    S, F, k = 64, 220, 96
    pair = Pair(S)
    scenes = [ts.scene(100 + s, F, objects=int(5 + (s % 8) * 4), k=k, clutter=2 + s % 3) for s in range(S)]
    pos = [0] * S
    rng = np.random.default_rng(1)
    empty = (np.zeros(k, np.float32), np.zeros(k, np.int32), np.zeros((k, 4), np.float32))
    for call in range(F):
        streams = [s for s in range(S) if rng.random() > 0.15]        # absent streams do not advance
        if call == 120:
            pair.reset([3, 17, 40])
        frames = []
        for s in streams:
            if s == 5 and call % 17 == 3:
                frames.append(empty)
            elif s == 6 and call % 13 == 4:
                frames.append(_all_low(k, rng))
            else:
                frames.append(scenes[s][pos[s]])
                pos[s] += 1
        rng.shuffle(streams_frames := list(zip(streams, frames)))
        pair.step([f for _, f in streams_frames], [s for s, _ in streams_frames], 64 if call % 5 else 7)
    pair.check_state()
    assert pair.outputs > 100000


@pytest.mark.parametrize("params", [dict(), dict(class_aware=1), dict(capacity=24, track_buffer=10), dict(fuse_score=0, match_thresh=0.9)])
def test_kernel_equals_spec_under_parameters(params):
    S, F, k = 8, 120, 128
    pair = Pair(S, **params)
    scenes = [ts.scene(200 + s, F, objects=30, k=k, ncls=2) for s in range(S)]
    for f in range(F):
        pair.step([scenes[s][f] for s in range(S)], list(range(S)), 128)
    pair.check_state()
    if "capacity" in params:
        assert all(st.overflow > 0 for st in pair.spec)


def test_exact_duplicate_entries_tie_in_the_assignment():
    S, F, k = 4, 60, 120
    pair = Pair(S)
    for f in range(F):
        frames = []
        for s in range(S):
            sc, lb, bx = ts.scene(300 + s, F, objects=20, k=60)[f]
            frames.append((np.r_[sc, sc], np.r_[lb, lb], np.r_[bx, bx]))   # every entry twice: equal costs everywhere
        pair.step(frames, list(range(S)), 120)
    pair.check_state()


@pytest.mark.parametrize("case", sorted(DUPLICATE_CASES))
def test_kernel_equals_spec_in_each_duplicate_case(case):
    """Every branch of step 8 on purpose: a younger lost track dropped, a younger tracked track dropped, the tie, a birth
    dropped at once (the kernel's TF_DROP and bdrop paths)."""
    frames, kw, survivors, dropped = DUPLICATE_CASES[case]
    pair = Pair(1, **kw)
    for f in frames:
        pair.step([ts.pad(*_frame(f), 4)], [0], 4)
    assert ([t.id for t in pair.spec[0].tracked], [t.id for t in pair.spec[0].lost]) == survivors
    assert pair.spec[0].dropped == dropped
    pair.check_state()


@pytest.mark.parametrize("kw", [dict(), dict(match_thresh=0.15)])
def test_kernel_equals_spec_on_scenes_with_many_duplicates(kw):
    """Echo detections start tracks on top of tracks, so step 8 drops tracked and lost tracks (and births at a low
    match_thresh) many times per stream."""
    S, F, k = 8, 160, 96
    pair = Pair(S, **kw)
    scenes = [ts.scene(400 + s, F, objects=12, k=k, occlusion=0.03, echo=0.08) for s in range(S)]
    for f in range(F):
        pair.step([scenes[s][f] for s in range(S)], list(range(S)), 96)
    pair.check_state()
    d = {key: sum(st.dropped[key] for st in pair.spec) for key in ("tracked", "birth", "lost")}
    assert d["tracked"] >= 20 and d["lost"] >= 20 and (d["birth"] >= 20 if kw else d["birth"] == 0), d


@pytest.mark.parametrize("spacing", [1.5, 4.0])
def test_crowd_frame_with_one_component_of_more_than_300_rows(spacing):
    """400 overlapping objects side by side drifting together: the first association is one component of 400 tracks.
    At 1.5 px spacing it has more admissible pairs than the kernel keeps (8192), so everything is solved as one component;
    at 4 px it has fewer, so the label propagation and the component sort find it."""
    k, n = 1024, 400
    pair = Pair(2, capacity=1024)
    rng = np.random.default_rng(4)
    cx = 500 + np.arange(n) * spacing
    pairs = []
    for f in range(12):
        cx = cx + 0.7
        w = np.full(n, 60.0) * (1 + rng.normal(0, 0.01, n))
        b = np.stack([cx - w / 2, 300 - 50 + rng.normal(0, 0.5, n), cx + w / 2, 300 + 50 + rng.normal(0, 0.5, n)], 1).astype(np.float32)
        s = rng.uniform(0.6, 0.95, n).astype(np.float32)
        frames = [ts.pad(s, np.zeros(n, np.int32), b, k), ts.pad(s[::-1].copy(), np.zeros(n, np.int32), b[::-1].copy(), k)]
        if f:                                           # the first association this frame will run, restated
            st = copy.deepcopy(pair.spec[0])
            pool = [t for t in st.tracked if t.activated] + st.lost
            for t in pool:
                ts.predict(t)
            cost = st._cost(pool, np.arange(n), st.p["match_thresh"], True, frames[0])
            rows, _ = ts.components(cost)
            assert max(len(r) for r in rows) >= 300
            pairs.append(int(np.isfinite(cost).sum()))
        pair.step(frames, [0, 1], 1024)
    assert min(pairs) > 8192 if spacing < 2 else max(pairs) < 8192, pairs
    pair.check_state()


def test_cuda_graph_of_the_three_calls_equals_eager():
    """forward_frames -> query_best -> track captured in one CUDA graph over a static frame buffer (the engine's plan made by
    a warm-up call, its own graphs off), replayed frame after frame, against the same calls run eagerly on a second tracker."""
    from b200 import capi
    model = _model()
    eng = model.engine()
    B = 4
    base = np.random.default_rng(3).integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)
    seq = [torch.from_numpy(np.roll(base, 3 * i, axis=2)).cuda() for i in range(8)]
    sizes = torch.tensor([[480.0, 640.0]] * B).cuda()

    def three(frames, tracker):
        out = eng.forward_frames(list(frames.unbind(0)), want_aux=False)
        s, l, b = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)
        return tracker.update(s, l, b, max_out=300)
    eager, graphed, probe = capi.Tracker(B, **LOW), capi.Tracker(B, **LOW), capi.Tracker(B, **LOW)
    want = [[t.cpu() for t in three(f, eager)] for f in seq]
    static = seq[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                         # warm-up outside the capture, on a third tracker
        three(static, probe)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = three(static, graphed)
    for i, f in enumerate(seq):
        static.copy_(f)
        graph.replay()
        for g_, w_ in zip(outs, want[i]):
            assert torch.equal(g_.cpu(), w_), i
    assert sum(int(w[5].sum()) for w in want) > 0
    got, want_state = graphed.export(0), eager.export(0)   # export waits for the replayed launches too
    assert got[1] == want_state[1] and got[1][0] == len(seq) + 1 and len(got[0]) == len(want_state[0]) > 0
    for x, y in zip(got[0], want_state[0]):
        for key in x:
            assert np.array_equal(np.asarray(x[key]), np.asarray(y[key])), key


def test_query_best_equals_postprocess_entries():
    from b200 import capi
    B, nq, ncls = 3, 100, 91
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(B, nq, ncls, generator=g) * 3).cuda()
    logits[0, 7, 10] = logits[0, 7, 20] = 9.0                   # an exact tie: the lower class
    boxes = torch.rand(B, nq, 4, generator=g).cuda()
    sizes = torch.tensor([[480.0, 640.0], [1080.0, 1920.0], [333.0, 517.0]]).cuda()
    s, l, b = capi.query_best(logits, boxes, sizes)
    ps, pl, pb = capi.postprocess(logits, boxes, sizes, nq * ncls)           # every (query, class) pair
    ts_ = torch.sigmoid(logits)
    assert torch.equal(l.long(), ts_.argmax(-1))
    assert l[0, 7] == 10
    for i in range(B):
        key = {(tuple(_bits(pb[i, j].cpu().numpy())), int(pl[i, j])): j for j in range(nq * ncls)}
        for q in range(nq):
            j = key[(tuple(_bits(b[i, q].cpu().numpy())), int(l[i, q]))]
            assert _bits(ps[i, j].cpu().numpy()) == _bits(s[i, q].cpu().numpy())


def _model():
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    return model.cuda()


LOW = dict(track_thresh=0.0, low_thresh=0.0, new_track_thresh=0.0)       # every query of the synthetic weights is "high"


def _by_hand(model, frames, streams, tracker, colorspace=None, max_out=300):
    from b200 import capi
    fb = capi.Frames(frames, colorspace=colorspace)
    out = model.engine().forward_frames(fb, want_aux=False)
    sizes = torch.tensor(fb.sizes, dtype=torch.float32, device="cuda")
    s, l, b = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)
    res, seen = [None] * len(streams), {}
    rounds = {}
    for i, st in enumerate(streams):
        rounds.setdefault(seen.get(st, 0), []).append(i)
        seen[st] = seen.get(st, 0) + 1
    for r in sorted(rounds):
        rows = rounds[r]
        idx = torch.tensor(rows, device="cuda")
        got = tracker.update(s[idx], l[idx], b[idx], [streams[i] for i in rows], max_out)
        for j, i in enumerate(rows):
            c = int(got[5][j])
            res[i] = {"ids": got[0][j, :c], "scores": got[1][j, :c], "labels": got[2][j, :c].long(), "boxes": got[3][j, :c],
                      "queries": got[4][j, :c].long()}
    return res


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for key in ("ids", "scores", "labels", "boxes", "queries"):
            assert torch.equal(g[key], w[key]), key


def test_track_equals_the_steps_composed_by_hand_with_several_frames_per_stream():
    from b200 import capi
    model = _model()
    rng = np.random.default_rng(9)
    base = [rng.integers(0, 256, (720, 1280, 3), dtype=np.uint8) for _ in range(3)]
    a, b = capi.Tracker(3, **LOW), capi.Tracker(3, **LOW)
    total = 0
    for call in range(3):
        frames, streams = [], [0, 1, 0, 2, 0, 1]                  # stream 0 three times, stream 1 twice in one call
        for i, st in enumerate(streams):
            f = np.roll(base[st], 4 * (call * 3 + i), axis=1)
            frames.append(torch.from_numpy(f).cuda())
        got = model.track(frames, a, streams=streams)
        want = _by_hand(model, frames, streams, b)
        _same(got, want)
        total += sum(int(g["ids"].numel()) for g in got)
    assert total > 0


def test_track_from_nv12_equals_rgb():
    from b200 import capi
    model = _model()
    rng = np.random.default_rng(7)
    packed = [rng.integers(0, 256, (720 * 3 // 2, 1280), dtype=np.uint8) for _ in range(2)]
    nv12 = [torch.from_numpy(p).cuda() for p in packed]
    rgb = [torch.from_numpy(yuv_spec.nv12_to_rgb(*yuv_spec.split_packed(p), "bt709")).cuda() for p in packed]
    a, b = capi.Tracker(2, **LOW), capi.Tracker(2, **LOW)
    for _ in range(2):
        got = model.track(nv12, a, colorspace="bt709")
        want = model.track(rgb, b)
        _same(got, want)
        assert got[0]["ids"].numel() > 0


def test_tracker_rejections():
    from b200 import capi
    t = capi.Tracker(2)
    z = torch.zeros(2, 4, device="cuda")
    zb = torch.zeros(2, 4, 4, device="cuda")
    with pytest.raises(RuntimeError, match="appears twice"):
        t.update(z, z.int(), zb, [1, 1])
    with pytest.raises(RuntimeError, match="outside"):
        t.update(z, z.int(), zb, [0, 2])
    with pytest.raises(RuntimeError, match="capacity"):
        capi.Tracker(1, capacity=2000)
    with pytest.raises(RuntimeError, match=r"\(0, 1\]"):
        capi.Tracker(1, match_thresh=1.5)
