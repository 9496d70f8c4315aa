"""GPU tests of tiled detection: the merge kernel (csrc/tiles.cu, lwdetr_tile_merge) bit for bit against its specification
(tools/tile_spec.py), and LWDETR.detect_tiled against the same steps composed by hand."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import tile_spec  # noqa: E402
import yuv_spec  # noqa: E402
from test_tiles_cpu import candidates, random_views  # noqa: E402


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


def _merge_both(scores, labels, boxes, views, F, score_threshold, thr, metric, max_det):
    from b200 import capi
    got = capi.tile_merge(torch.from_numpy(scores).cuda(), torch.from_numpy(labels).cuda(), torch.from_numpy(boxes).cuda(), views, F,
                          score_threshold, thr, metric, max_det)
    torch.cuda.synchronize()
    want = tile_spec.merge(scores, labels, boxes, views, F, score_threshold, thr, metric, max_det)
    for name, g, w in zip(("scores", "labels", "boxes", "counts"), got, want):
        assert np.array_equal(_bits(g.cpu().numpy()), _bits(w)), name
    return want


@pytest.mark.parametrize("metric", ["ios", "iou"])
def test_kernel_equals_spec_on_frames_with_different_view_counts(metric):
    counts = [9, 33, 1, 5]
    views = random_views(1, counts)
    scores, labels, boxes = candidates(1, len(views), 100, ncls=6, span=600.0)
    want = _merge_both(scores, labels, boxes, views, len(counts), 0.0, 0.5, metric, 300)
    assert all(want[3] > 0)


@pytest.mark.parametrize("metric", ["ios", "iou"])
def test_kernel_equals_spec_on_heavy_overlap_with_exact_ties(metric):
    counts = [6, 3]
    views = [(f, 0, 0) for f, c in enumerate(counts) for _ in range(c)]         # every view at the origin: maximal overlap
    scores, labels, boxes = candidates(2, len(views), 300, ncls=2, span=40.0, wh=(20.0, 60.0), ties=True)
    for thr in (0.3, 0.5, 0.9):
        want = _merge_both(scores, labels, boxes, views, len(counts), 0.0, thr, metric, 1000)
        assert 0 < want[3].min()
        if thr <= 0.5:
            assert want[3].max() < 900                                         # most of the 1800 / 900 are suppressed


@pytest.mark.parametrize("metric", ["ios", "iou"])
def test_kernel_equals_spec_with_degenerate_boxes_and_an_empty_frame(metric):
    counts = [4, 3, 0, 2]                                                      # frame 2 has no view at all
    views = random_views(3, counts)
    scores, labels, boxes = candidates(3, len(views), 64, span=100.0, degenerate=0.2)
    scores[4:7] *= 0.4                                                         # frame 1: nothing reaches the threshold
    want = _merge_both(scores, labels, boxes, views, len(counts), 0.45, 0.5, metric, 300)
    assert want[3][1] == 0 and want[3][2] == 0 and want[3][0] > 0


def test_kernel_stops_at_max_det():
    views = random_views(4, [8, 2])
    scores, labels, boxes = candidates(4, len(views), 100, ncls=20, span=3000.0)
    for max_det in (1, 17, 300):
        want = _merge_both(scores, labels, boxes, views, 2, 0.0, 0.5, "ios", max_det)
        assert want[3][0] == max_det


def test_kernel_at_16384_candidates_in_one_frame():
    views = random_views(5, [128, 3])                                          # frame 0: 128 views x 128 = 16384
    scores, labels, boxes = candidates(5, len(views), 128, ncls=8, span=400.0)
    for metric in ("ios", "iou"):
        want = _merge_both(scores, labels, boxes, views, 2, 0.0, 0.5, metric, 1024)
        assert want[3][0] == 1024


@pytest.mark.parametrize("per_frame", [1, 2, 3])
def test_kernel_with_one_candidate_per_view(per_frame):
    """k = 1: with one view per frame the shared key region is at its smallest, and the kept list after it must stay
    16-byte aligned."""
    counts = [per_frame] * 7
    views = random_views(8, counts)
    scores, labels, boxes = candidates(8, len(views), 1, ncls=2, span=30.0)
    for metric in ("ios", "iou"):
        want = _merge_both(scores, labels, boxes, views, len(counts), 0.0, 0.5, metric, 5)
        assert (want[3] >= 1).all()


def test_kernel_over_several_launches():
    """600 frames and 3000 views: more frames and views than one launch carries."""
    counts = [(f % 9) + 1 for f in range(600)]
    views = random_views(6, counts)
    scores, labels, boxes = candidates(6, len(views), 4, ncls=3, span=200.0)
    _merge_both(scores, labels, boxes, views, len(counts), 0.1, 0.5, "iou", 20)


def test_kernel_rejects_beyond_its_limits():
    from b200 import capi
    z = lambda V, k: (torch.zeros(V, k, device="cuda"), torch.zeros(V, k, device="cuda", dtype=torch.int32),
                      torch.zeros(V, k, 4, device="cuda"))
    for (V, k), views, F, kw, msg in (((1, 16385), [(0, 0, 0)], 1, {}, "16384 candidates"),
                                      ((2049, 1), [(0, 0, 0)] * 2049, 1, {}, "2048 views"),
                                      ((2, 10), [(0, 0, 0), (0, 0, 0)], 1, dict(max_det=1025), r"\[1, 1024\]"),
                                      ((2, 10), [(0, 0, 0), (0, 0, 0)], 1, dict(max_det=0), r"\[1, 1024\]"),
                                      ((2, 10), [(1, 0, 0), (0, 0, 0)], 2, {}, "non-decreasing"),
                                      ((2, 10), [(0, 0, 0), (2, 0, 0)], 2, {}, "outside"),
                                      ((2, 10), [(0, 0, 0), (0, 0, 0)], 1, dict(iou_threshold=1.5), r"\[0, 1\]")):
        with pytest.raises(RuntimeError, match=msg):
            capi.tile_merge(*z(V, k), views, F, **kw)
    with pytest.raises(RuntimeError, match="metric"):
        capi.tile_merge(*z(1, 1), [(0, 0, 0)], 1, metric="giou")
    # the limits themselves run: 16384 zero boxes (degenerate: nothing suppresses) with equal scores -> the first 1024 by flat index
    s, l, b, c = capi.tile_merge(*z(128, 128), [(0, 0, 0)] * 128, 1, max_det=1024)
    torch.cuda.synchronize()
    assert c.item() == 1024 and (l == 0).all() and (s == 0).all() and (b == 0).all()


# ----------------------------------------------------------------------------------------------- composition
def _noise(h, w, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8))


def _model():
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    return model.cuda()


def _by_hand(model, frames, kw):
    """tile_views -> forward_frames on the crop views with their dsts (one batch) -> capi.postprocess -> tile_spec.merge."""
    from b200 import capi
    from b200.config import tile_views
    from models.lwdetr import tile_crops
    fb = capi.Frames(frames, colorspace=kw.get("colorspace"))
    per_view = kw.get("per_view", 100)
    (H, W), views = tile_views(model.cfg, fb.sizes, kw.get("tile"), kw.get("overlap", 0.2), kw.get("full_frame", True), kw.get("size"),
                               per_view)
    out = model.engine().forward_frames(tile_crops(fb, views), size=(H, W), dsts=[(v[5], v[6]) for v in views], want_aux=False)
    sizes = torch.tensor([(v[3], v[4]) for v in views], dtype=torch.float32, device="cuda")
    s, l, b = capi.postprocess(out["pred_logits"], out["pred_boxes"], sizes, per_view)
    torch.cuda.synchronize()
    return views, tile_spec.merge(s.cpu().numpy(), l.cpu().numpy(), b.cpu().numpy(), [(v[0], v[2], v[1]) for v in views],
                                  len(fb.items), kw.get("score_threshold", 0.0), kw.get("iou_threshold", 0.5),
                                  kw.get("metric", "ios"), kw.get("max_det", 300))


def _same(det, want):
    s, l, b, c = want
    assert len(det) == len(c)
    for f, d in enumerate(det):
        n = int(c[f])
        assert d["scores"].shape == (n,) and d["labels"].dtype == torch.int64 and d["boxes"].shape == (n, 4)
        assert np.array_equal(_bits(d["scores"].cpu().numpy()), _bits(s[f, :n]))
        assert np.array_equal(d["labels"].cpu().numpy(), l[f, :n])
        assert np.array_equal(_bits(d["boxes"].cpu().numpy()), _bits(b[f, :n]))


@pytest.mark.parametrize("kw", [dict(), dict(metric="iou", iou_threshold=0.6, score_threshold=0.05, max_det=100, per_view=50)])
def test_detect_tiled_equals_the_steps_composed_by_hand(kw):
    model = _model()
    frames = [_noise(1080, 1920, 1).cuda(), _noise(2160, 3840, 2).cuda()]
    views, want = _by_hand(model, frames, kw)
    assert len(views) == 9 + 33
    _same(model.detect_tiled(frames, **kw), want)
    assert (want[3] > 0).all()
    model.engine().set_option("cuda_graph", 1)
    for _ in range(3):                         # eager first run of the plan, then graph capture, then replay
        _same(model.detect_tiled(frames, **kw), want)


def test_detect_tiled_partial_tiles_and_a_small_frame():
    """A frame smaller than the tile on one axis (partial tiles, padded and masked) and one smaller on both, with tile
    (480, 800) on a 448 x 768 run size."""
    model = _model()
    frames = [_noise(400, 2000, 3).cuda(), _noise(300, 500, 4).cuda()]
    kw = dict(tile=(480, 800), size=(448, 768))
    views, want = _by_hand(model, frames, kw)
    assert views[0][5:] == (373, 768) and views[-2][5:] == (280, 480)
    _same(model.detect_tiled(frames, **kw), want)


def test_detect_tiled_one_detection_per_view():
    """per_view = 1 without the full view on frames no larger than the tile: one candidate per frame reaches the merge."""
    model = _model()
    frames = [_noise(480, 640, 5).cuda(), _noise(300, 500, 6).cuda(), _noise(640, 640, 7).cuda()]
    kw = dict(per_view=1, full_frame=False)
    views, want = _by_hand(model, frames, kw)
    assert len(views) == 3 and (want[3] == 1).all()
    _same(model.detect_tiled(frames, **kw), want)


def test_detect_tiled_from_nv12_equals_rgb():
    """NV12 frames (a packed 1080p one and (luma, chroma) planes of odd sizes) against the RGB frames yuv_spec converts them
    to: the crops sit at even offsets, so every view sees exactly the same pixels."""
    model = _model()
    rng = np.random.default_rng(7)
    packed = rng.integers(0, 256, (1080 * 3 // 2, 1920), dtype=np.uint8)
    odd_y = rng.integers(0, 256, (1081, 1917), dtype=np.uint8)
    odd_c = rng.integers(0, 256, (541, 2 * 959), dtype=np.uint8)
    nv12 = [torch.from_numpy(packed).cuda(), (torch.from_numpy(odd_y).cuda(), torch.from_numpy(odd_c).cuda())]
    rgb = [torch.from_numpy(yuv_spec.nv12_to_rgb(*yuv_spec.split_packed(packed), "bt709")).cuda(),
           torch.from_numpy(yuv_spec.nv12_to_rgb(odd_y, odd_c, "bt709")).cuda()]
    got = model.detect_tiled(nv12, colorspace="bt709")
    want = model.detect_tiled(rgb)
    for g, w in zip(got, want):
        assert g["scores"].numel() > 0
        for key in ("scores", "labels", "boxes"):
            assert torch.equal(g[key], w[key]), key


def test_forward_frames_dsts_rejections():
    model = _model()
    eng = model.engine()
    z = torch.zeros(64, 64, 3, dtype=torch.uint8, device="cuda")
    for kw, msg in ((dict(dsts=[(64, 64)], fit="keep_aspect", short_side=64), "do not combine"),
                    (dict(dsts=[(64, 64), (64, 64)]), "2 dsts for 1 frames"), (dict(dsts=[(641, 64)]), "does not fit"),
                    (dict(dsts=[(0, 64)]), "does not fit")):
        with pytest.raises(RuntimeError, match=msg):
            eng.forward_frames([z], **kw)
