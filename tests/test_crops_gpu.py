"""GPU tests of the detection crops (lwdetr_crops / _nv12, lwdetr_crop_select, lwdetr_scatter_rows; csrc/crops.cu) against
tools/crop_spec.py: levels equal except at tie pixels, normalised values equal to normalise() of the kernel's levels in each
output dtype; a device count; select and scatter against torch; a CUDA graph of select -> crops -> scatter; and
LWDETR.track(reid=) against track(appearance=) fed with the same network's rows."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import crop_spec  # noqa: E402
import resize_spec  # noqa: E402
import yuv_spec  # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def _rgb_frame(h, w, rng, pad=7, off=5):
    """A CUDA RGB frame [h, w, 3] inside a larger buffer: row pitch 3w + pad, first pixel `off` bytes in."""
    buf = torch.from_numpy(rng.integers(0, 256, (h + 1) * (3 * w + pad) + off, dtype=np.uint8)).cuda()
    return torch.as_strided(buf, (h, w, 3), (3 * w + pad, 3, 1), off)


def _nv12_frame(h, w, rng, pad=9, off=3):
    """(luma, chroma) CUDA planes with padded pitches at odd offsets."""
    cw = 2 * ((w + 1) // 2)
    lb = torch.from_numpy(rng.integers(0, 256, (h, w + pad + off), dtype=np.uint8)).cuda()
    cb = torch.from_numpy(rng.integers(0, 256, ((h + 1) // 2, cw + pad + off), dtype=np.uint8)).cuda()
    return lb[:, off:off + w], cb[:, off:off + cw]


def _host_rgb(frames, nv12, cs):
    if not nv12:
        return [f.cpu().numpy() for f in frames]
    return crop_spec.nv12_frames([(y.cpu().numpy(), c.cpu().numpy()) for y, c in frames], [cs] * len(frames))


def _boxes(rng, sizes, n):
    """Random boxes over the frames, plus 1x1 crops, crops past the edges and invalid ones."""
    out, fidx = [], []
    for i in range(n):
        f = int(rng.integers(0, len(sizes)))
        h, w = sizes[f]
        kind = i % 8
        if kind == 0:
            x, y = rng.uniform(0, w - 1), rng.uniform(0, h - 1)
            b = [x, y, np.floor(x) + 1.5, np.floor(y) + 1.2]                     # a 1 x 1 crop
        elif kind == 1:
            b = [rng.uniform(-50, w / 2), rng.uniform(-50, h / 2), rng.uniform(w / 2, w + 50), rng.uniform(h / 2, h + 50)]
        elif kind == 2:
            b = [[np.nan, 1, 5, 5], [w + 1, 0, w + 9, 9], [5, 5, 5.5, 20], [1, 1, np.inf, 9]][i // 8 % 4]
        else:
            x0, y0 = rng.uniform(0, w - 2), rng.uniform(0, h - 2)
            b = [x0, y0, x0 + rng.uniform(1, min(w - x0, 400)), y0 + rng.uniform(1, min(h - y0, 600))]
        out.append(b)
        fidx.append(f)
    return np.array(out, np.float32), np.array(fidx, np.int32)


def _check(frames, nv12, boxes, fidx, size, filter, cs="bt709", dtypes=("fp32",)):
    from b200 import capi
    fb = capi.Frames(frames, colorspace=cs if nv12 else None)
    host = _host_rgb(frames, nv12, cs)
    bt, ft = torch.from_numpy(boxes).cuda(), torch.from_numpy(fidx).cuda()
    lv, valid = capi.crops(fb, bt, ft, size, filter, normalize=False)
    _, want_u8, want_raw, want_valid = crop_spec.crops(host, boxes, fidx, size, filter, normalize=False)
    assert np.array_equal(valid.cpu().numpy(), want_valid)
    got = lv.cpu().numpy()
    assert np.array_equal(got, np.floor(got)) and got.min() >= 0 and got.max() <= 255
    ties = resize_spec.tie_pixels(want_raw)
    bad = (got != want_u8) & ~ties
    assert not bad.any(), ("levels differ off tie pixels", int(bad.sum()), np.argwhere(bad)[:5])
    assert np.abs(got - want_u8).max() <= 1
    assert not got[~want_valid].any()
    u8 = got.astype(np.uint8).transpose(0, 2, 3, 1)
    want_norm = torch.from_numpy(resize_spec.normalise(u8, MEAN, STD).transpose(0, 3, 1, 2).copy())
    want_norm[torch.from_numpy(~want_valid)] = 0
    for name in dtypes:
        out, _ = capi.crops(fb, bt, ft, size, filter, MEAN, STD, dtype=DTYPES[name])
        assert out.dtype == DTYPES[name]
        assert torch.equal(out.cpu(), want_norm.to(DTYPES[name])), name
    return int(want_valid.sum()), int(ties.sum())


@pytest.mark.parametrize("filter", ["bilinear", "antialias"])
@pytest.mark.parametrize("nv12", [False, True])
def test_kernel_equals_spec_odd_sizes_pitches_and_offsets(filter, nv12):
    rng = np.random.default_rng(11 + nv12 * 2 + (filter == "antialias"))
    sizes = [(257, 391), (480, 640), (9, 11)]
    frames = [_nv12_frame(h, w, rng) if nv12 else _rgb_frame(h, w, rng) for h, w in sizes]
    boxes, fidx = _boxes(rng, sizes, 96)
    for size in ((37, 19), (256, 128), (8, 1024)):
        nvalid, nties = _check(frames, nv12, boxes, fidx, size, filter, dtypes=("fp32", "fp16", "bf16"))
        print("%s %s %s: %d valid crops, %d tie values" % (filter, "nv12" if nv12 else "rgb", size, nvalid, nties))
        assert nvalid > 60


def test_whole_4k_frame_to_8x8_antialias():
    rng = np.random.default_rng(12)
    for nv12 in (False, True):
        frames = [_nv12_frame(2160, 3840, rng) if nv12 else _rgb_frame(2160, 3840, rng)]
        boxes = np.array([[0, 0, 3840, 2160], [-10, -10, 1e9, 1e9], [1.5, 3.5, 3001.2, 2001.7]], np.float32)
        _check(frames, nv12, boxes, np.zeros(3, np.int32), (8, 8), "antialias", dtypes=("fp16",))


def test_more_frames_and_crops_than_one_launch_group():
    rng = np.random.default_rng(13)
    sizes = [(int(rng.integers(8, 60)), int(rng.integers(8, 60))) for _ in range(150)]
    for nv12 in (False, True):
        frames = [_nv12_frame(h, w, rng) if nv12 else _rgb_frame(h, w, rng) for h, w in sizes]
        boxes, fidx = _boxes(rng, sizes, 3000)
        fidx[:3] = [-1, 150, 7]                                  # a frame index outside [0, B) is an invalid crop
        _check(frames, nv12, boxes, fidx, (16, 8), "bilinear")


def test_device_count_leaves_rows_past_it_untouched():
    from b200 import capi
    rng = np.random.default_rng(14)
    frames = [_rgb_frame(100, 120, rng) for _ in range(2)]
    boxes, fidx = _boxes(rng, [(100, 120)] * 2, 12)
    bt, ft = torch.from_numpy(boxes).cuda(), torch.from_numpy(fidx).cuda()
    ref, ref_valid = capi.crops(frames, bt, ft, (16, 8), dtype=torch.float16)
    out = torch.full((12, 3, 16, 8), 1234.0, device="cuda", dtype=torch.float16)
    valid = torch.full((12,), 7, device="cuda", dtype=torch.int8)
    capi.crops(frames, bt, ft, (16, 8), dtype=torch.float16, count=torch.tensor([5], device="cuda"), out=out, valid=valid)
    assert torch.equal(out[:5], ref[:5]) and torch.equal(valid[:5].bool(), ref_valid[:5])
    assert (out[5:] == 1234.0).all() and (valid[5:] == 7).all()


def _torch_select(scores, boxes, sizes, thr):
    """Restatement in torch of lwdetr_crop_select: (frame, entry, boxes) of the kept entries in (frame, entry) order."""
    B, k = scores.shape
    hw = torch.tensor(sizes, dtype=torch.float32, device=scores.device)
    x0, y0, x1, y1 = (torch.floor(boxes[..., i]) for i in range(4))
    W, H = hw[:, 1:2], hw[:, 0:1]
    cx0, cx1 = torch.minimum(torch.clamp(x0, min=0), W), torch.minimum(torch.clamp(x1, min=0), W)
    cy0, cy1 = torch.minimum(torch.clamp(y0, min=0), H), torch.minimum(torch.clamp(y1, min=0), H)
    keep = (scores > thr) & torch.isfinite(boxes).all(-1) & (cx1 > cx0) & (cy1 > cy0)
    flat = torch.nonzero(keep.flatten()).flatten()
    return (flat // k).int(), flat.int(), boxes.reshape(-1, 4)[flat]


def test_select_and_scatter_equal_torch_and_replay_under_a_graph():
    from b200 import capi
    rng = np.random.default_rng(15)
    B, k, D = 70, 40, 24                                           # two select launch groups
    sizes = [(int(rng.integers(50, 300)), int(rng.integers(50, 300))) for _ in range(B)]
    frames = [_rgb_frame(h, w, rng) for h, w in sizes]
    scores = torch.from_numpy(rng.uniform(0, 1, (B, k)).astype(np.float32)).cuda()
    bx = np.stack([_boxes(rng, [s], k)[0] for s in sizes])
    boxes = torch.from_numpy(bx).cuda()
    scores[3, :] = float("nan")
    fr, en, sb, cnt = capi.crop_select(scores, boxes, sizes, 0.3)
    wf, we, wb = _torch_select(scores, boxes, sizes, 0.3)
    c = int(cnt.item())
    assert c == wf.numel() > 0
    assert torch.equal(fr[:c], wf) and torch.equal(en[:c], we) and torch.equal(sb[:c], wb)
    want_sel = crop_spec.select(scores.cpu().numpy(), bx, sizes, 0.3)
    assert [e for _, e, _ in want_sel] == en[:c].cpu().tolist()
    rows = torch.randn(c, D + 3, device="cuda", dtype=torch.bfloat16)[:, :D]
    got = capi.scatter_rows(rows, en[:c], B * k)
    want = torch.zeros(B * k, D, device="cuda", dtype=torch.bfloat16)
    want[we.long()] = rows
    assert torch.equal(got, want)
    # select -> crops (N = B * k, device count) -> scatter of a fixed-size row block, captured once and replayed
    N = B * k
    fb = capi.Frames(frames)
    proj = torch.randn(3 * 16 * 8, D, device="cuda")

    def step():
        f, e, b, n = capi.crop_select(scores, boxes, sizes, 0.3)
        cr, va = capi.crops(fb, b, f, (16, 8), count=n, out=out, valid=val)
        r = cr.reshape(N, -1) @ proj
        return capi.scatter_rows(r, e, B * k, count=n), va
    out = torch.zeros(N, 3, 16, 8, device="cuda")
    val = torch.zeros(N, device="cuda", dtype=torch.int8)
    eager, eva = (t.clone() for t in step())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    out.zero_()
    val.zero_()
    with torch.cuda.graph(g):
        res, rva = step()
    out.zero_()
    val.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(res, eager) and torch.equal(rva, eva)
    assert res.abs().sum() > 0


class _Reid(torch.nn.Module):
    """A small deterministic CNN standing in for a ReID network."""

    def __init__(self, D):
        super().__init__()
        torch.manual_seed(0)
        self.net = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, stride=2), torch.nn.ReLU(), torch.nn.AdaptiveAvgPool2d(1),
                                       torch.nn.Flatten(), torch.nn.Linear(8, D))
        self.calls = 0

    def forward(self, x):
        self.calls += 1
        return self.net(x)


def _appearance_of(model, fb, m, thr, size):
    """T [frames, nq, D]: capi.crops of the high entries with a valid crop, m, scattered by torch."""
    from b200 import capi
    out = model.engine().forward_frames(fb, want_aux=False)
    sizes = torch.tensor(fb.sizes, dtype=torch.float32, device="cuda")
    scores, _, boxes = capi.query_best(out["pred_logits"], out["pred_boxes"], sizes)
    n, nq = scores.shape
    flat = torch.nonzero((scores > thr).flatten()).flatten()
    crops, valid = capi.crops(fb, boxes.reshape(-1, 4)[flat], flat // nq, size)
    with torch.no_grad():
        rows = m(crops[valid])
    T = torch.zeros(n * nq, rows.shape[1], device="cuda")
    T[flat[valid]] = rows
    return T.view(n, nq, -1)


@pytest.mark.parametrize("nv12", [False, True])
def test_track_with_reid_equals_track_with_its_embeddings(nv12):
    from b200 import capi
    from test_track_gpu import LOW, _model
    model = _model()
    D = 16
    m = _Reid(D).cuda().eval()
    rng = np.random.default_rng(16)
    cs = "bt709" if nv12 else None
    for motion in (False, True):
        for streams in ([0, 1, 2], [0, 0, 1]):
            a, b = capi.Tracker(3, embedding_dim=D, **LOW), capi.Tracker(3, embedding_dim=D, **LOW)
            ga, gb = (capi.MotionEstimator(3), capi.MotionEstimator(3)) if motion else (None, None)
            for call in range(3):
                frames = [_nv12_frame(360, 640, rng) if nv12 else _rgb_frame(360, 640, rng) for _ in range(3)]
                fb = capi.Frames(frames, colorspace=cs)
                calls = m.calls
                x = model.track(fb, a, streams=streams, motion=ga, reid=m, reid_size=(64, 32))
                assert m.calls == calls + 1
                T = _appearance_of(model, fb, m, float(a.params.track_thresh), (64, 32))
                y = model.track(fb, b, streams=streams, motion=gb, appearance=T)
                for g, w in zip(x, y):
                    for key in g:
                        assert torch.equal(g[key], w[key]), key
            for s in range(3):
                ea, ha = a.export_embeddings(s)
                eb, hb = b.export_embeddings(s)
                assert np.array_equal(ha, hb) and np.array_equal(ea[ha], eb[hb])
            assert any(a.export_embeddings(s)[1].any() for s in range(3))


def test_track_with_reid_and_no_crops_does_not_call_the_network():
    from b200 import capi
    from test_track_gpu import _model
    model = _model()
    m = _Reid(16).cuda().eval()
    t = capi.Tracker(2, embedding_dim=16, track_thresh=1.0, low_thresh=0.0, new_track_thresh=1.0)
    rng = np.random.default_rng(17)
    model.track([_rgb_frame(200, 300, rng) for _ in range(2)], t, reid=m)
    assert m.calls == 0


def test_rejections():
    from b200 import capi
    from test_track_gpu import _model
    rng = np.random.default_rng(18)
    fr = [_rgb_frame(40, 50, rng)]
    b, f = torch.zeros(1, 4, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match=r"\[8, 1024\]"):
        capi.crops(fr, b, f, (4, 8))
    with pytest.raises(RuntimeError, match=r"\[8, 1024\]"):
        capi.crops(fr, b, f, (8, 2048))
    with pytest.raises(RuntimeError, match="filter"):
        capi.crops(fr, b, f, (8, 8), "nearest")
    with pytest.raises(RuntimeError, match="std must be positive"):
        capi.crops(fr, b, f, (8, 8), std=(1.0, 0.0, 1.0))
    with pytest.raises(RuntimeError, match="dtype"):
        capi.crops(fr, b, f, (8, 8), dtype=torch.float64)
    with pytest.raises(RuntimeError, match=r"sides must be in \[8, 8192\]"):
        capi.crops([_rgb_frame(4, 50, rng)], b, f, (8, 8))
    big = torch.zeros(65537, 4, device="cuda")
    with pytest.raises(RuntimeError, match=r"N must be in \[1, 65536\]"):
        capi.crops(fr, big, torch.zeros(65537, dtype=torch.int32, device="cuda"), (8, 8))
    with pytest.raises(RuntimeError, match="NaN"):
        capi.crop_select(torch.zeros(1, 2, device="cuda"), torch.zeros(1, 2, 4, device="cuda"), [(10, 10)], float("nan"))
    model = _model()
    t = capi.Tracker(1, embedding_dim=16)
    m = _Reid(16).cuda().eval()
    with pytest.raises(RuntimeError, match="not both"):
        model.track(fr, t, reid=m, appearance=True)
    with pytest.raises(RuntimeError, match="embedding_dim"):
        model.track(fr, capi.Tracker(1), reid=m)
    with pytest.raises(RuntimeError, match=r"\[\d+, 8\]"):
        model.track(fr, capi.Tracker(1, embedding_dim=8, track_thresh=0.0, low_thresh=0.0), reid=m)


def test_model_crops_from_detect():
    from test_track_gpu import _model
    model = _model()
    rng = np.random.default_rng(19)
    frames = [_rgb_frame(300, 400, rng), _rgb_frame(120, 90, rng)]
    dets = model.detect(frames, num_select=20)
    crops, frame = model.crops(frames, dets, (32, 16), dtype=torch.float16)
    assert crops.shape == (40, 3, 32, 16) and frame.tolist() == [0] * 20 + [1] * 20
    host = _host_rgb(frames, False, None)
    boxes = torch.cat([d["boxes"] for d in dets]).cpu().numpy()
    want = crop_spec.crops(host, boxes, frame.cpu().numpy(), (32, 16), "bilinear", MEAN, STD)
    from b200 import capi
    lv, _ = capi.crops(frames, torch.from_numpy(boxes).cuda(), frame, (32, 16), normalize=False)
    ties = resize_spec.tie_pixels(want[2])
    assert not ((lv.cpu().numpy() != want[1]) & ~ties).any()
