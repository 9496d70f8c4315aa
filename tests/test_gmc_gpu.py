"""GPU tests of camera-motion compensation: the estimator's kernels (csrc/gmc.cu) against their specification
(tools/gmc_spec.py) and OpenCV, its accuracy on frames with a known motion against BoT-SORT's method, determinism and CUDA
graphs; lwdetr_track_ex against the tracker specification with the true camera motion; LWDETR.track(motion=...) against
the same steps composed by hand."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gmc_spec as gs  # noqa: E402
import track_spec as ts  # noqa: E402

cv2 = pytest.importorskip("cv2")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.view(np.int64) if a.dtype == np.float64 else a


def _rgb_view(img, pad):
    """A CUDA RGB frame whose rows are 3 * (w + pad) bytes apart."""
    h, w, _ = img.shape
    big = torch.zeros(h, w + pad, 3, dtype=torch.uint8, device="cuda")
    big[:, :w] = torch.from_numpy(img).cuda()
    return big[:, :w]


def _nv12_view(luma, chroma, pad):
    h, w = luma.shape
    y = torch.zeros(h, w + pad, dtype=torch.uint8, device="cuda")
    y[:, :w] = torch.from_numpy(luma).cuda()
    c = torch.zeros(chroma.shape[0], chroma.shape[1] + pad, dtype=torch.uint8, device="cuda")
    c[:, :chroma.shape[1]] = torch.from_numpy(chroma).cuda()
    return (y[:, :w], c[:, :chroma.shape[1]])


def _odd_nv12(rgb):
    """Luma of an RGB frame of any size (the estimator reads only it) and a chroma plane of the NV12 shape."""
    h, w, _ = rgb.shape
    luma = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV)[..., 0].copy()
    return luma, np.full(((h + 1) // 2, 2 * ((w + 1) // 2)), 128, np.uint8)


@pytest.mark.parametrize("fmt", ["rgb", "nv12"])
@pytest.mark.parametrize("size,pad", [((479, 637), 3), ((480, 640), 0), ((1080, 1920), 1), ((203, 333), 5)])
def test_pyramid_and_corners_equal_the_specification(fmt, size, pad):
    from b200 import capi
    h, w = size
    p = gs.params()
    est = capi.MotionEstimator(2)
    rgb = gs.textured_frame(h + w, h, w)
    if fmt == "rgb":
        frames, grey = [_rgb_view(rgb, pad)], gs.grey_rgb(rgb)
    else:
        luma, chroma = _odd_nv12(rgb)
        frames, grey = [_nv12_view(luma, chroma, pad)], luma
    est.estimate(frames, [1])
    got = est.export(1)
    want = gs.pyramid(grey, p)
    assert got["valid"] and got["size"] == (h, w) and len(got["levels"]) == len(want)
    for l, (a, b) in enumerate(zip(got["levels"], want)):
        assert np.array_equal(a, b), l
    wc = gs.corners(want[0], p)
    print("%s %dx%d: %d corners, 0 differing (responses compared exactly, no ties within 1 ulp to excuse)" % (fmt, h, w, len(wc)))
    assert len(wc) > 50 and np.array_equal(got["corners"], wc)


def test_lucas_kanade_agrees_with_opencv():
    from b200 import capi
    p = gs.params()
    truth = gs.similarity(1.5, 1.03, 17.0, -9.0, (640, 360))
    prev, cur, _ = gs.moving_pair(5, 720, 1280, truth)
    est = capi.MotionEstimator(1)
    est.estimate([torch.from_numpy(prev).cuda()])
    est.estimate([torch.from_numpy(cur).cuda()])
    st = est.export(0)
    a, b = gs.level0(gs.grey_rgb(prev), 2), gs.level0(gs.grey_rgb(cur), 2)
    pts = st["flow"][:, :2].copy()
    assert np.array_equal(pts, gs.corners(a, p))
    nxt, status, _ = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), None, winSize=(21, 21), maxLevel=3)
    both = st["found"] & (status.reshape(-1) == 1)
    d = np.sqrt(((st["flow"][both, 2:] - nxt.reshape(-1, 2)[both]) ** 2).sum(1))
    frac = float((d <= 0.05).mean())
    print("LK: %d points, %d found by both, %.4f within 0.05 px, max %.3f px; found only by one: %d"
          % (len(pts), both.sum(), frac, d.max(), int((st["found"] != (status.reshape(-1) == 1)).sum())))
    assert both.sum() > 0.8 * len(pts) and frac >= 0.95


SIZES = {"480p": (480, 640), "1080p": (1080, 1920), "4k": (2160, 3840)}


@pytest.mark.parametrize("fmt", ["rgb", "nv12"])
@pytest.mark.parametrize("res", list(SIZES))
def test_estimator_accuracy_against_botsort(res, fmt):
    from b200 import capi
    h, w = SIZES[res]
    rng = np.random.default_rng(len(res) * 10 + len(fmt))
    est = capi.MotionEstimator(1)
    worst, worst_ref = 0.0, 0.0
    for trial in range(3):
        truth = gs.similarity(rng.uniform(-3, 3), rng.uniform(0.95, 1.05), rng.uniform(-40, 40), rng.uniform(-40, 40),
                              (w / 2, h / 2))
        prev, cur, _ = gs.moving_pair(100 * trial + h, h, w, truth)
        if fmt == "rgb":
            fr = [[torch.from_numpy(prev).cuda()], [torch.from_numpy(cur).cuda()]]
            ref = gs.botsort_gmc(prev, cur)
        else:
            (yp, cp), (yc, cc) = gs.rgb_to_nv12(prev), gs.rgb_to_nv12(cur)
            fr = [[(torch.from_numpy(yp).cuda(), torch.from_numpy(cp).cuda())], [(torch.from_numpy(yc).cuda(), torch.from_numpy(cc).cuda())]]
            ref = gs.botsort_gmc(yp, yc)
        est.reset([0])
        m0, s0, _ = est.estimate(fr[0])
        m, s, inl = est.estimate(fr[1])
        assert int(s0[0]) == capi.GMC_FIRST_FRAME and int(s[0]) == capi.GMC_OK
        e = gs.corner_error(m[0].cpu().numpy(), truth, h, w)
        er = gs.corner_error(ref, truth, h, w)
        print("%s %s trial %d: corner error %.3f px (BoT-SORT's method %.3f px), %d inliers" % (res, fmt, trial, e, er, int(inl[0])))
        worst, worst_ref = max(worst, e), max(worst_ref, er)
        assert e <= 0.5 and e <= 1.5 * er + 0.1, (e, er)
    print("%s %s: worst corner error %.3f px, BoT-SORT's method %.3f px" % (res, fmt, worst, worst_ref))


def test_statuses_first_frame_size_change_textureless_and_reset():
    from b200 import capi
    est = capi.MotionEstimator(3)
    a = torch.from_numpy(gs.textured_frame(1, 480, 640)).cuda()
    b = torch.from_numpy(gs.textured_frame(2, 360, 640)).cuda()
    flat = torch.full((480, 640, 3), 90, dtype=torch.uint8, device="cuda")
    ident = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64)

    def call(frames, streams):
        m, s, i = est.estimate(frames, streams)
        return m.cpu(), s.cpu().tolist(), i.cpu().tolist()
    m, s, _ = call([a, flat, a], [0, 1, 2])
    assert s == [capi.GMC_FIRST_FRAME] * 3 and all(torch.equal(x, ident) for x in m)
    m, s, _ = call([b, flat, a], [0, 1, 2])
    assert s == [capi.GMC_SIZE_CHANGED, capi.GMC_FEW_POINTS, capi.GMC_OK] and torch.equal(m[0], ident) and torch.equal(m[1], ident)
    est.reset([2])
    m, s, i = call([a], [2])
    assert s == [capi.GMC_FIRST_FRAME] and i == [0] and torch.equal(m[0], ident)
    m, s, i = call([b], [0])
    assert s == [capi.GMC_OK] and i[0] > 100 and np.allclose(m[0].numpy(), [1, 0, 0, 0], atol=1e-6)
    with pytest.raises(RuntimeError, match="appears twice"):
        est.estimate([a, a], [1, 1])
    with pytest.raises(RuntimeError, match="outside"):
        est.estimate([a], [3])
    with pytest.raises(RuntimeError, match="sides must be"):
        est.estimate([torch.zeros(20, 640, 3, dtype=torch.uint8, device="cuda")], [0])
    with pytest.raises(RuntimeError, match="window"):
        capi.MotionEstimator(1, window=20)


def _sequence(n, h, w, seed, camera=None):
    """n RGB frames of one textured scene seen through a camera path (true motion per frame)."""
    motion = ts.camera_path(n, (h, w), **(camera or dict(ts.CAMERA, seed=seed)))
    big = gs.textured_frame(seed, h, w, margin=200)
    acc = np.array([1.0, 0.0, 0.0, 0.0])
    out = []
    for f in range(n):
        a, b, tx, ty = motion[f]
        acc = np.array([a * acc[0] - b * acc[1], b * acc[0] + a * acc[1], (a * acc[2] - b * acc[3]) + tx, (b * acc[2] + a * acc[3]) + ty])
        view = gs.matrix(acc) @ np.array([[1, 0, -200], [0, 1, -200], [0, 0, 1.0]])
        out.append(cv2.warpAffine(big, view, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101))
    return out, motion


def test_two_runs_are_bit_identical():
    from b200 import capi
    frames, _ = _sequence(6, 720, 1280, 3)
    res = []
    for _ in range(2):
        est = capi.MotionEstimator(4)
        got = []
        for f in frames:
            batch = [torch.from_numpy(np.roll(f, 13 * s, axis=1)).cuda() for s in range(4)]
            got.append([t.cpu().numpy() for t in est.estimate(batch, [3, 0, 2, 1])])
        res.append(got)
    for x, y in zip(*res):
        for u, v in zip(x, y):
            assert np.array_equal(_bits(u), _bits(v))
    assert all(int(s) == 0 for x in res[0][1:] for s in x[1])


def test_cuda_graph_of_estimate_and_track_equals_eager():
    from b200 import capi
    B, n = 3, 8
    seqs = [_sequence(n, 480, 640, 40 + s)[0] for s in range(B)]
    dets = [ts.scene(60 + s, n, objects=15, k=64) for s in range(B)]

    def step(est, trk, frames, sc, lb, bx):
        m, s, i = est.estimate(frames, list(range(B)))
        return (m, s, i) + trk.update(sc, lb, bx, motion=m)

    def inputs(f):
        return ([torch.from_numpy(seqs[s][f]).cuda() for s in range(B)],
                torch.from_numpy(np.stack([dets[s][f][0] for s in range(B)])).cuda(),
                torch.from_numpy(np.stack([dets[s][f][1] for s in range(B)])).cuda(),
                torch.from_numpy(np.stack([dets[s][f][2] for s in range(B)])).cuda())
    e_est, e_trk = capi.MotionEstimator(B), capi.Tracker(B)
    want = [[t.cpu() for t in step(e_est, e_trk, *inputs(f))] for f in range(n)]
    g_est, g_trk = capi.MotionEstimator(B), capi.Tracker(B)
    w_est, w_trk = capi.MotionEstimator(B), capi.Tracker(B)
    static = [x.clone() for x in inputs(0)[0]]
    sc, lb, bx = (x.clone() for x in inputs(0)[1:])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(w_est, w_trk, static, sc, lb, bx)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step(g_est, g_trk, static, sc, lb, bx)
    for f in range(n):
        fr, s2, l2, b2 = inputs(f)
        for d, x in zip(static, fr):
            d.copy_(x)
        sc.copy_(s2)
        lb.copy_(l2)
        bx.copy_(b2)
        graph.replay()
        for g_, w_ in zip(outs, want[f]):
            assert torch.equal(g_.cpu(), w_), f
    assert all(int(x) == 0 for w in want[1:] for x in w[1])


@pytest.mark.parametrize("streams,class_aware", [(1, 0), (32, 0), (32, 1), (256, 0), (256, 1)])
def test_track_ex_with_true_motion_equals_the_specification(streams, class_aware):
    from b200 import capi
    F = {1: 200, 32: 80, 256: 24}[streams]
    k = 64
    kw = dict(class_aware=class_aware)
    dev = capi.Tracker(streams, **kw)
    spec = [ts.Stream(ts.params(**kw)) for _ in range(streams)]
    scenes = [ts.scene(500 + s, F, objects=12 + s % 10, k=k, ncls=2, camera=dict(ts.CAMERA, seed=s)) for s in range(streams)]
    outs = 0
    for f in range(F):
        sc = torch.from_numpy(np.stack([scenes[s][0][f][0] for s in range(streams)])).cuda()
        lb = torch.from_numpy(np.stack([scenes[s][0][f][1] for s in range(streams)])).cuda()
        bx = torch.from_numpy(np.stack([scenes[s][0][f][2] for s in range(streams)])).cuda()
        mo = torch.from_numpy(np.stack([scenes[s][1][f] for s in range(streams)])).cuda()
        got = [g.cpu().numpy() for g in dev.update(sc, lb, bx, max_out=k, motion=mo)]
        for s in range(streams):
            want = ts.outputs_array(spec[s].update(*scenes[s][0][f], motion=scenes[s][1][f]), k)
            for name, g, w in zip(("ids", "scores", "labels", "boxes", "index", "count"), got, want):
                assert np.array_equal(_bits(g[s]), _bits(np.asarray(w))), (s, f, name)
            outs += want[5]
    for s in range(streams):
        recs, fno = dev.export(s)
        want = spec[s].export()
        assert fno == (spec[s].frame, spec[s].next_id, spec[s].overflow) and len(recs) == len(want)
        for g, w in zip(recs, want):
            assert np.array_equal(_bits(g["mean"]), _bits(w["mean"])) and np.array_equal(_bits(g["cov"]), _bits(w["cov"])), s
    assert outs > 5 * streams * F


def test_track_ex_with_null_motion_is_track():
    from b200 import capi
    S, F, k = 16, 60, 96
    a, b = capi.Tracker(S), capi.Tracker(S)
    scenes = [ts.scene(700 + s, F, objects=20, k=k) for s in range(S)]
    ids = (ctypes.c_int32 * S)(*range(S))
    for f in range(F):
        sc = torch.from_numpy(np.stack([scenes[s][f][0] for s in range(S)])).cuda()
        lb = torch.from_numpy(np.stack([scenes[s][f][1] for s in range(S)])).cuda()
        bx = torch.from_numpy(np.stack([scenes[s][f][2] for s in range(S)])).cuda()
        want = a.update(sc, lb, bx, max_out=k)
        got = [torch.empty_like(t) for t in want]
        capi.check(capi.lib().lwdetr_track_ex(b._t, capi.ptr(sc), capi.ptr(lb), capi.ptr(bx), None, S, k, ctypes.cast(ids, ctypes.c_void_p), k,
                                              *[capi.ptr(t) for t in got], capi.stream_ptr(b.device)), "lwdetr_track_ex")
        for g, w in zip(got, want):
            assert torch.equal(g, w), f
    for s in range(S):
        x, y = a.export(s), b.export(s)
        assert x[1] == y[1] and len(x[0]) == len(y[0])
        for u, v in zip(x[0], y[0]):
            assert np.array_equal(u["mean"], v["mean"]) and np.array_equal(u["cov"], v["cov"])


LOW = dict(track_thresh=0.0, low_thresh=0.0, new_track_thresh=0.0)       # every query of the synthetic weights is "high"


def _model():
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    return model.cuda()


@pytest.mark.parametrize("fmt", ["rgb", "nv12"])
def test_model_track_with_motion_equals_the_steps_composed_by_hand(fmt):
    from b200 import capi
    model = _model()
    S, n = 32, 3
    seqs = [_sequence(n, 360, 640, 80 + s % 4, dict(ts.CAMERA, seed=s))[0] for s in range(S)]
    cs = None if fmt == "rgb" else "bt601"

    def frames(f):
        if fmt == "rgb":
            return [torch.from_numpy(seqs[s][f]).cuda() for s in range(S)]
        return [tuple(torch.from_numpy(x).cuda() for x in gs.rgb_to_nv12(seqs[s][f])) for s in range(S)]
    streams = list(range(S))[::-1]
    ta, tb = capi.Tracker(S, **LOW), capi.Tracker(S, **LOW)
    ea, eb = capi.MotionEstimator(S, max_height=360, max_width=640), capi.MotionEstimator(S, max_height=360, max_width=640)
    total = 0
    for f in range(n):
        fr = frames(f)
        got = model.track(fr, ta, streams=streams, colorspace=cs, motion=ea)
        fb = capi.Frames(fr, colorspace=cs)
        out = model.engine().forward_frames(fb, want_aux=False)
        sizes = torch.tensor(fb.sizes, dtype=torch.float32, device="cuda")
        s_, l_, b_ = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)
        m, st, _ = eb.estimate(fb, streams)
        if f:
            assert all(int(x) == 0 for x in st.cpu())
        want = tb.update(s_, l_, b_, streams, model.num_queries, motion=m)
        for i in range(S):
            c = int(want[5][i])
            w = {"ids": want[0][i, :c], "scores": want[1][i, :c], "labels": want[2][i, :c].long(), "boxes": want[3][i, :c],
                 "queries": want[4][i, :c].long()}
            for key in w:
                assert torch.equal(got[i][key], w[key]), (f, i, key)
            total += c
    assert total > 0
