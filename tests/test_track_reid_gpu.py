"""GPU tests of tracking by appearance (lwdetr_track_reid, the appearance instantiation of csrc/track.cu) bit for bit
against its specification (tools/track_spec.py with reid_params()): outputs every frame, then the float64 records and
the fp32 track embeddings via export; lwdetr_last_hidden against class_embed and the oracle's decoder output; LWDETR.track
with appearance against the specification fed with the same hidden state."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402
from test_track_gpu import LOW, _bits, _model  # noqa: E402

DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


class ReidPair:
    """A device tracker with appearance and one specification stream per stream id, driven together."""

    def __init__(self, num_streams, dim, reid=None, **params):
        from b200 import capi
        reid = dict(reid or {})
        self.dim = dim
        self.dev = capi.Tracker(num_streams, embedding_dim=dim, **reid, **params)
        self.spec = [ts.Stream(ts.params(**params), ts.reid_params(embedding_dim=dim, **reid)) for _ in range(num_streams)]
        self.outputs = 0

    def reset(self, streams):
        self.dev.reset(streams)
        for s in streams:
            self.spec[s].reset()

    def step(self, frames, embs, streams, max_out, dtype="fp32", pad=0, motion=None, raw=None):
        """frames: per stream id in `streams`, (scores, labels, boxes) of one common k; embs: float32 [k, dim] each (or
        None: the call passes no embeddings); pad: extra elements per row (row stride dim + pad).  raw: "lwdetr_track" or
        "lwdetr_track_ex" called directly through the C ABI instead of Tracker.update (embs None)."""
        sc = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
        lb = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
        bx = torch.from_numpy(np.stack([f[2] for f in frames])).cuda()
        emb = None
        if embs is not None:
            B, k = sc.shape
            full = torch.zeros(B, k, self.dim + pad, dtype=DTYPES[dtype])
            full[..., :self.dim] = torch.from_numpy(np.stack(embs)).to(DTYPES[dtype])
            emb = full.cuda()[..., :self.dim]
        mo = None if motion is None else torch.from_numpy(np.stack(motion)).cuda()
        if raw is None:
            got = [g.cpu().numpy() for g in self.dev.update(sc, lb, bx, streams, max_out, motion=mo, embeddings=emb)]
        else:
            assert emb is None
            got = [g.cpu().numpy() for g in _raw(self.dev, raw, sc, lb, bx, mo, streams, max_out)]
        spec_emb = None if emb is None else emb.float().cpu().numpy()
        for r, (s, f) in enumerate(zip(streams, frames)):
            want = ts.outputs_array(self.spec[s].update(*f, motion=None if motion is None else motion[r],
                                                        embeddings=None if spec_emb is None else spec_emb[r]), max_out)
            for name, g, w in zip(("ids", "scores", "labels", "boxes", "index", "count"), got, want):
                assert np.array_equal(_bits(g[r]), _bits(np.asarray(w))), "stream %d frame %d: %s" % (s, self.spec[s].frame - 1, name)
            self.outputs += want[5]

    def check_state(self):
        n_emb = 0
        for s, spec in enumerate(self.spec):
            recs, fno = self.dev.export(s)
            assert fno == (spec.frame, spec.next_id, spec.overflow), s
            want = spec.export()
            assert [g["id"] for g in recs] == [w["id"] for w in want], s
            for g, w in zip(recs, want):
                assert np.array_equal(_bits(g["mean"]), _bits(w["mean"])) and np.array_equal(_bits(g["cov"]), _bits(w["cov"])), s
            emb, has = self.dev.export_embeddings(s)
            want_e = spec.export_embeddings()
            assert list(has) == [e is not None for e in want_e], s
            for g, w in zip(emb, want_e):
                if w is not None:
                    assert np.array_equal(_bits(g), _bits(w)), s
                    n_emb += 1
        return n_emb


def _raw(tracker, name, sc, lb, bx, mo, streams, max_out):
    """lwdetr_track / lwdetr_track_ex through the C ABI on a tracker made with appearance."""
    import ctypes
    from b200 import capi
    B, k = sc.shape
    outs = [torch.empty(B, max_out, dtype=torch.int32, device="cuda"), torch.empty(B, max_out, device="cuda"),
            torch.empty(B, max_out, dtype=torch.int32, device="cuda"), torch.empty(B, max_out, 4, device="cuda"),
            torch.empty(B, max_out, dtype=torch.int32, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")]
    ids = (ctypes.c_int32 * B)(*streams)
    args = [tracker._t, capi.ptr(sc), capi.ptr(lb), capi.ptr(bx)] + ([capi.ptr(mo)] if name == "lwdetr_track_ex" else [])
    args += [B, k, ctypes.cast(ids, ctypes.c_void_p), max_out] + [capi.ptr(o) for o in outs] + [capi.stream_ptr()]
    capi.check(getattr(capi.lib(), name)(*args), name)
    return outs


def _scenes(S, F, k, dim, seed0, **kw):
    out = []
    for s in range(S):
        frames, motion, _, embs = ts.scene(seed0 + s, F, objects=int(6 + (s % 6) * 4), k=k, clutter=2 + s % 3, crossings=3,
                                           appearance=dict(seed=seed0 + s, dim=dim, cosine=0.85), **kw)
        out.append((frames, motion, embs))
    return out


def _spoil(e, rng):
    """Some rows zero and some with a NaN: those entries have no appearance."""
    e = e.copy()
    e[rng.random(len(e)) < 0.05] = 0.0
    e[rng.random(len(e)) < 0.05, 0] = np.nan
    return e


def test_64_streams_with_absent_streams_resets_zero_and_nan_rows_fp16_strided():
    S, F, k, D = 64, 120, 96, 100
    pair = ReidPair(S, D)
    scenes = _scenes(S, F, k, D, 500)
    pos = [0] * S
    rng = np.random.default_rng(2)
    for call in range(F):
        streams = [s for s in range(S) if rng.random() > 0.15]
        if call == 60:
            pair.reset([3, 17, 40])
        frames = [scenes[s][0][pos[s]] for s in streams]
        embs = [_spoil(scenes[s][2][pos[s]], rng) for s in streams]
        for s in streams:
            pos[s] += 1
        pair.step(frames, embs, streams, 64, dtype="fp16", pad=12)
    assert pair.check_state() > 500
    assert pair.outputs > 20000


@pytest.mark.parametrize("dim, dtype, pad", [(64, "fp32", 0), (256, "bf16", 8), (256, "fp32", 3), (2048, "fp16", 0)])
def test_kernel_equals_spec_across_dims_and_dtypes(dim, dtype, pad):
    S, F, k = 8 if dim < 2048 else 4, 80, 128
    pair = ReidPair(S, dim)
    scenes = _scenes(S, F, k, dim, 600)
    for f in range(F):
        pair.step([sc[0][f] for sc in scenes], [sc[2][f] for sc in scenes], list(range(S)), 128, dtype=dtype, pad=pad)
    assert pair.check_state() > 8 * S


@pytest.mark.parametrize("S", [1, 32])
@pytest.mark.parametrize("params", [dict(), dict(class_aware=1), dict(fuse_score=0, match_thresh=0.9)])
def test_kernel_equals_spec_with_motion_and_parameters(S, params):
    F, k, D = 80, 96, 64
    pair = ReidPair(S, D, reid=dict(appearance_thresh=0.3, ema_alpha=0.8), **params)
    scenes = _scenes(S, F, k, D, 700, camera=dict(ts.CAMERA, seed=3))
    for f in range(F):
        pair.step([sc[0][f] for sc in scenes], [sc[2][f] for sc in scenes], list(range(S)), 96, motion=[sc[1][f] for sc in scenes])
    assert pair.check_state() > 4 * S


def _proximity_pairs(st, boxes, prox=0.5):
    """(record, high entry) pairs within proximity, both with appearance, as the kernel lists them before association 1:
    every record with an embedding (confirmed and lost ones predicted, unconfirmed ones not) x the given entries (all high,
    all with appearance)."""
    tb = []
    for t in st.tracked + st.lost:
        if t.emb is None:
            continue
        t2 = ts.Track()
        t2.p, t2.v, t2.P, t2.C, t2.V, t2.state = t.p.copy(), t.v.copy(), t.P.copy(), t.C.copy(), t.V.copy(), t.state
        if t.activated or t.state == ts.LOST:
            ts.predict(t2)
        tb.append(t2.box())
    if not tb:
        return 0
    io = ts.iou(np.array(tb), boxes.astype(np.float64))
    return int((1.0 - io <= np.float64(np.float32(prox))).sum())


@pytest.mark.parametrize("spacing", [1.5, 4.0])
def test_crowd_with_more_proximity_pairs_than_the_table_holds(spacing):
    """400 objects side by side: at 1.5 px spacing the first association has more than 8192 proximity pairs (and more than
    8192 admissible pairs), so the lanes compute the appearance costs themselves inside the one-component solve; at 4 px
    the pair table holds them."""
    k, n, D = 1024, 400, 64
    pair = ReidPair(2, D, reid=dict(appearance_thresh=0.4), capacity=1024)
    rng = np.random.default_rng(4)
    cx = 500 + np.arange(n) * spacing
    u = rng.normal(size=(n, D))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    counts = []
    for f in range(10):
        cx = cx + 0.7
        w = np.full(n, 60.0) * (1 + rng.normal(0, 0.01, n))
        b = np.stack([cx - w / 2, 300 - 50 + rng.normal(0, 0.5, n), cx + w / 2, 300 + 50 + rng.normal(0, 0.5, n)], 1).astype(np.float32)
        s = rng.uniform(0.6, 0.95, n).astype(np.float32)
        e = (u + rng.normal(0, 0.3, (n, D))).astype(np.float32)
        ep = np.zeros((k, D), np.float32)
        ep[:n] = e
        er = np.zeros((k, D), np.float32)
        er[:n] = e[::-1]
        if f:                                           # the pairs the kernel lists this frame, per stream
            counts += [_proximity_pairs(st, b) for st in pair.spec]
        pair.step([ts.pad(s, np.zeros(n, np.int32), b, k), ts.pad(s[::-1].copy(), np.zeros(n, np.int32), b[::-1].copy(), k)], [ep, er],
                  [0, 1], 1024)
    assert min(counts) > 8192 if spacing < 2 else max(counts) < 8192, counts
    pair.check_state()


def test_track_and_track_ex_mixed_with_track_reid_on_one_tracker():
    """lwdetr_track and lwdetr_track_ex on a tracker made with appearance run as lwdetr_track_reid without embeddings: the
    tracks keep their embeddings and slots, so the calls can alternate with lwdetr_track_reid (births in the plain calls
    have no embedding until a reid update gives them one)."""
    S, F, k, D = 16, 90, 96, 64
    pair = ReidPair(S, D)
    scenes = _scenes(S, F, k, D, 1000, camera=dict(ts.CAMERA, seed=7))
    for f in range(F):
        frames = [sc[0][f] for sc in scenes]
        motion = [sc[1][f] for sc in scenes]
        if f % 3 == 0:
            pair.step(frames, [sc[2][f] for sc in scenes], list(range(S)), 96, motion=motion)
        elif f % 3 == 1:
            pair.step(frames, None, list(range(S)), 96, motion=motion, raw="lwdetr_track_ex")
        else:                                          # no motion: the still-camera call on a moving scene is fine here
            pair.step(frames, None, list(range(S)), 96, raw="lwdetr_track")
    n = pair.check_state()
    assert n > 4 * S
    assert any(e is None for st in pair.spec for e in st.export_embeddings())


def test_null_embeddings_equal_track_ex():
    from b200 import capi
    S, F, k = 16, 60, 96
    scenes = _scenes(S, F, k, 32, 800, camera=dict(ts.CAMERA, seed=5))
    a, b = capi.Tracker(S, embedding_dim=32), capi.Tracker(S)
    for f in range(F):
        sc = torch.from_numpy(np.stack([x[0][f][0] for x in scenes])).cuda()
        lb = torch.from_numpy(np.stack([x[0][f][1] for x in scenes])).cuda()
        bx = torch.from_numpy(np.stack([x[0][f][2] for x in scenes])).cuda()
        mo = torch.from_numpy(np.stack([x[1][f] for x in scenes])).cuda()
        for g, w in zip(a.update(sc, lb, bx, motion=mo), b.update(sc, lb, bx, motion=mo)):
            assert torch.equal(g, w), f
    for s in range(S):
        x, y = a.export(s), b.export(s)
        assert x[1] == y[1] and [r["id"] for r in x[0]] == [r["id"] for r in y[0]]
        assert not a.export_embeddings(s)[1].any()


def test_cuda_graph_replay_equals_eager():
    from b200 import capi
    S, F, k, D = 8, 40, 96, 64
    scenes = _scenes(S, F, k, D, 900)
    args = [(torch.from_numpy(np.stack([x[0][f][0] for x in scenes])).cuda(),
             torch.from_numpy(np.stack([x[0][f][1] for x in scenes])).cuda(),
             torch.from_numpy(np.stack([x[0][f][2] for x in scenes])).cuda(),
             torch.from_numpy(np.stack([x[2][f] for x in scenes])).cuda().half()) for f in range(F)]
    eager, graphed, probe = (capi.Tracker(S, embedding_dim=D) for _ in range(3))
    want = [[t.cpu() for t in eager.update(*a_[:3], embeddings=a_[3])] for a_ in args]
    static = [t.clone() for t in args[0]]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        probe.update(*static[:3], embeddings=static[3])
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = graphed.update(*static[:3], embeddings=static[3])
    for f in range(F):
        for d_, s_ in zip(static, args[f]):
            d_.copy_(s_)
        graph.replay()
        for g_, w_ in zip(outs, want[f]):
            assert torch.equal(g_.cpu(), w_), f
    for s in range(S):
        x, y = graphed.export_embeddings(s), eager.export_embeddings(s)
        assert np.array_equal(x[1], y[1]) and np.array_equal(_bits(x[0]), _bits(y[0]))
    assert sum(int(w[5].sum()) for w in want) > 0


def test_last_hidden_is_the_layer_class_embed_reads():
    from b200.config import CONFIGS
    from b200.synth import synth_images, synth_state_dict
    from oracle import lwdetr_oracle as orc
    import torch.nn.functional as Fn
    cfg = CONFIGS["tiny"]
    sd = synth_state_dict(cfg, 1)
    model = _model()
    rng = np.random.default_rng(11)
    frames = [torch.from_numpy(rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)).cuda() for _ in range(2)]
    out = model.engine().forward_frames(frames, want_aux=False, want_hidden=True)
    h = out["hidden"]
    assert h.shape == (2, cfg.num_queries, cfg.hidden_dim) and h.dtype == torch.float16
    # class_embed as the engine holds it (fp16 weight, fp32 bias), in float64: only the GEMM's fp32 accumulation differs
    W, bias, hd = sd["class_embed.weight"].half().double(), sd["class_embed.bias"].double(), h.cpu().double()
    logits = Fn.linear(hd, W, bias)
    scale = Fn.linear(hd.abs(), W.abs(), bias.abs())          # sum of |terms| per logit
    err = ((logits - out["pred_logits"].cpu().double()).abs() / scale).max().item()
    print("hidden through class_embed vs pred_logits: max error %.3e of the sum of |terms|" % err)
    assert err < 1e-5, err
    # against the oracle's last decoder layer (after the decoder's norm), top-k forced to the oracle's
    x = synth_images(1, 0)
    inter = {}
    orc.forward(sd, cfg, x, inter=inter)
    key = [n for n in sd if n.endswith("decoder.norm.weight")][0]
    want = Fn.layer_norm(inter["dec%d" % (cfg.dec_layers - 1)], (cfg.hidden_dim,), sd[key], sd[key.replace("weight", "bias")], 1e-5)
    eng = model.engine()
    eng.forward(x.cuda(), want_aux=False, topk_override=inter["topk"])
    got = torch.empty(1, cfg.num_queries, cfg.hidden_dim + 8, device="cuda", dtype=torch.float16)
    from b200 import capi
    capi.check(capi.lib().lwdetr_last_hidden(eng._h, capi.ptr(got), cfg.hidden_dim + 8, capi.stream_ptr()), "lwdetr_last_hidden")
    got = got[..., :cfg.hidden_dim].float().cpu()
    rel = ((got - want).norm() / want.norm()).item()
    print("last hidden vs oracle: rel-L2 %.3e" % rel)
    assert rel < 1e-2, rel


def _spec_track(model, frames, streams, specs, hidden_of, colorspace=None):
    """The specification fed with forward_frames -> query_best and the given per-frame embeddings."""
    from b200 import capi
    fb = capi.Frames(frames, colorspace=colorspace)
    out = model.engine().forward_frames(fb, want_aux=False, want_hidden=True)
    sizes = torch.tensor(fb.sizes, dtype=torch.float32, device="cuda")
    s, l, b = (t.cpu().numpy() for t in capi.query_best(out["pred_logits"], out["pred_boxes"], sizes))
    emb = hidden_of(out).float().cpu().numpy()
    return [ts.outputs_array(specs[st].update(s[i], l[i], b[i], embeddings=emb[i]), 300) for i, st in enumerate(streams)]


def _check(got, want):
    for g, w in zip(got, want):
        c = w[5]
        assert g["ids"].numel() == c
        for key, x in zip(("ids", "scores", "labels", "boxes", "queries"), w[:5]):
            assert np.array_equal(_bits(g[key].cpu().numpy().astype(np.asarray(x).dtype)), _bits(np.asarray(x)[:c])), key


def test_track_with_appearance_equals_the_spec_fed_with_the_same_hidden_state():
    from b200 import capi
    model = _model()
    d = model.cfg.hidden_dim
    rng = np.random.default_rng(9)
    base = [rng.integers(0, 256, (720, 1280, 3), dtype=np.uint8) for _ in range(3)]
    tracker = capi.Tracker(3, embedding_dim=d, **LOW)
    specs = [ts.Stream(ts.params(**LOW), ts.reid_params(embedding_dim=d)) for _ in range(3)]
    total = 0
    for call in range(4):
        frames = [torch.from_numpy(np.roll(base[i], 5 * call, axis=1)).cuda() for i in range(3)]
        got = model.track(frames, tracker, max_out=300, appearance=True)
        want = _spec_track(model, frames, range(3), specs, lambda o: o["hidden"])
        _check(got, want)
        total += sum(w[5] for w in want)
    assert total > 0 and any(has.any() for has in (tracker.export_embeddings(s)[1] for s in range(3)))
    with pytest.raises(RuntimeError, match="embedding_dim"):
        model.track(frames, capi.Tracker(3, embedding_dim=d + 1), appearance=True)


def test_track_with_own_embeddings_and_motion_from_nv12_and_rgb():
    from b200 import capi
    import yuv_spec
    model = _model()
    rng = np.random.default_rng(7)
    packed = [rng.integers(0, 256, (720 * 3 // 2, 1280), dtype=np.uint8) for _ in range(2)]
    nv12 = [torch.from_numpy(p).cuda() for p in packed]
    rgb = [torch.from_numpy(yuv_spec.nv12_to_rgb(*yuv_spec.split_packed(p), "bt709")).cuda() for p in packed]
    nq = model.num_queries
    own = torch.randn(2, nq, 48, device="cuda")
    a, b = capi.Tracker(2, embedding_dim=48, **LOW), capi.Tracker(2, embedding_dim=48, **LOW)
    ga, gb = capi.MotionEstimator(2), capi.MotionEstimator(2)
    for _ in range(3):
        x = model.track(nv12, a, colorspace="bt709", appearance=own, motion=ga)
        y = model.track(rgb, b, appearance=own, motion=gb)
        for g, w in zip(x, y):
            for key in g:
                assert torch.equal(g[key], w[key]), key
        assert x[0]["ids"].numel() > 0
    assert a.export_embeddings(0)[1].any()
    c = capi.Tracker(2, embedding_dim=model.cfg.hidden_dim, **LOW)
    assert len(model.track(rgb, c, appearance=True, motion=capi.MotionEstimator(2))) == 2


def test_reid_rejections():
    from b200 import capi
    with pytest.raises(RuntimeError, match=r"\[1, 2048\]"):
        capi.Tracker(1, embedding_dim=4096)
    with pytest.raises(RuntimeError, match=r"\[0, 1\)"):
        capi.Tracker(1, embedding_dim=8, proximity_thresh=1.0)
    with pytest.raises(RuntimeError, match="without embedding_dim"):
        capi.Tracker(1, ema_alpha=0.5)
    t = capi.Tracker(2, embedding_dim=8)
    z = torch.zeros(2, 4, device="cuda")
    with pytest.raises(RuntimeError, match=r"\[2, 4, 8\]"):
        t.update(z, z.int(), torch.zeros(2, 4, 4, device="cuda"), embeddings=torch.zeros(2, 4, 7, device="cuda"))
    with pytest.raises(RuntimeError, match="embedding_dim"):
        capi.Tracker(2).update(z, z.int(), torch.zeros(2, 4, 4, device="cuda"), embeddings=torch.zeros(2, 4, 8, device="cuda"))
