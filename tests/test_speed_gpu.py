"""GPU tests of speed estimation: the kernel (csrc/speed.cu, lwdetr_speed_update) bit for bit against its specification
(tools/speed_spec.py) on device-tracker outputs for 1, 32 and 256 streams: kin, samples and every export field, with
changing stream subsets, set and reset mid-sequence, timestamps NULL and given, capacity and window at their limits and
max_out 1024; one CUDA graph of Tracker.update + Zones.update + SpeedEstimator.update replayed; an export that waits for
the object's own work only; LWDETR.track(speed=) against the specification run on the tracks it returned; rejections."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import speed_spec as sp  # noqa: E402
import track_spec as ts  # noqa: E402
import zone_spec as zs  # noqa: E402


def _same(a, b):
    """Bit-for-bit equality of float arrays, NaNs in the same places."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


class Pair:
    """A device speed object and one specification stream per stream id, driven together."""

    def __init__(self, num_streams, **params):
        from b200 import capi
        self.dev = capi.SpeedEstimator(num_streams, **params)
        self.spec = [sp.Stream(sp.params(**params)) for _ in range(num_streams)]
        self.estimates = 0

    def set(self, s, H):
        self.dev.set(s, H)
        self.spec[s].set(H)

    def reset(self, streams):
        self.dev.reset(streams)
        for s in streams:
            self.spec[s].reset()

    def update(self, ids, boxes, counts, streams, timestamps=None):
        kin, samples = self.dev.update(ids, boxes, counts, streams, timestamps)
        kin, samples = kin.cpu().numpy(), samples.cpu().numpy()
        ids, boxes, counts = [t.cpu().numpy() for t in (ids, boxes, counts)]
        ts_host = None if timestamps is None else np.asarray(timestamps.cpu() if torch.is_tensor(timestamps) else timestamps)
        for b, s in enumerate(streams):
            w_kin, w_n = self.spec[s].update(ids[b], boxes[b], counts[b], None if ts_host is None else ts_host[b])
            assert _same(kin[b], w_kin), (s, kin[b][:8], w_kin[:8])
            assert np.array_equal(samples[b], w_n), s
            self.estimates += int(np.isfinite(w_kin[:, 4]).sum())

    def compare_exports(self, streams=None):
        for s in range(len(self.spec)) if streams is None else streams:
            got, want = self.dev.export(s), self.spec[s].export()
            assert got.keys() == want.keys()
            for k in want:
                if k == "samples":
                    assert len(got[k]) == len(want[k]) and all(_same(g, w) for g, w in zip(got[k], want[k])), s
                else:
                    assert _same(got[k], want[k]), (s, k, got[k], want[k])


def tracked(S, frames, seed=0, objects=25, max_out=64):
    """Device-tracker outputs over seeded scenes, one per stream: a list per frame of (ids, boxes, counts) [S, ...]."""
    from b200 import capi
    k = 96
    scenes = [ts.scene(seed + s, frames, objects=objects, k=k, crossings=3) for s in range(S)]
    trk = capi.Tracker(S)
    out = []
    for f in range(frames):
        sc, lab, bx = (torch.from_numpy(np.stack([scenes[s][f][i] for s in range(S)])).cuda() for i in range(3))
        ids, _, _, boxes, _, counts = trk.update(sc, lab, bx, max_out=max_out)
        out.append((ids, boxes, counts))
    return out


def _camera_h(s):
    """A per-stream ground homography: the pinhole camera of speed_spec at a stream-dependent height and pitch."""
    return sp.camera(height=6.0 + s % 7, pitch_deg=15.0 + 3 * (s % 5))["H"]


@pytest.mark.parametrize("S,frames", [(1, 60), (32, 24), (256, 8)])
def test_kernel_equals_spec_with_subsets_set_reset_and_clocks(S, frames):
    rng = np.random.default_rng(S)
    pair = Pair(S, forget_after=4, capacity=40, window=8, min_samples=3)
    for s in range(0, S, 2):
        pair.set(s, _camera_h(s))
    clock = np.zeros(S)
    for f, (ids, boxes, counts) in enumerate(tracked(S, frames, seed=100)):
        rows = np.sort(rng.choice(S, size=max(1, int(rng.integers(S // 2, S + 1))), replace=False)) if S > 1 and f % 3 else np.arange(S)
        rng.shuffle(rows)
        idx = torch.from_numpy(rows).cuda()
        stamps = None
        if f % 2:                                   # given timestamps: mostly increasing, some stale or NaN
            clock[rows] += rng.uniform(0.02, 0.05, len(rows))
            st = clock[rows].copy()
            st[rng.random(len(rows)) < 0.1] = np.nan
            st[rng.random(len(rows)) < 0.1] -= 1.0
            stamps = torch.from_numpy(st).cuda()
        pair.update(ids[idx], boxes[idx], counts[idx], rows.tolist(), stamps)
        if f == frames // 2:
            pair.reset([int(x) for x in rows[: max(1, len(rows) // 4)]])
            pair.set(int(rows[-1]), _camera_h(1000 + f))
    pair.compare_exports()
    assert pair.estimates > 0


def test_capacity_window_and_max_out_at_the_limits():
    pair = Pair(2, capacity=4096, window=64, min_samples=64, forget_after=2)
    rng = np.random.default_rng(9)
    for s in range(2):
        pair.set(s, _camera_h(s))
    n = 1024
    for f in range(70):
        ids = np.zeros((2, n), np.int32)
        ids[:, :1000] = rng.permutation(np.arange(1, 1001 + 40 * f))[:1000].astype(np.int32) if f % 10 == 9 else np.arange(1, 1001)
        cx, cy = rng.uniform(0, 1920, (2, n)), rng.uniform(500, 1080, (2, n))
        boxes = np.stack([cx - 20, cy - 80, cx + 20, cy], -1).astype(np.float32)
        counts = np.array([1000, 1024], np.int32)
        pair.update(*(torch.from_numpy(x).cuda() for x in (ids, boxes, counts)), [0, 1])
    pair.compare_exports()
    assert pair.dev.export(0)["records"] > 1000
    tiny = Pair(1, capacity=1, window=2, min_samples=2)
    for ids, boxes, counts in tracked(1, 20, seed=3):
        tiny.update(ids, boxes, counts, [0])
    tiny.compare_exports()
    assert tiny.dev.export(0)["overflow"] > 0


def test_cuda_graph_of_track_zones_and_speed_equals_eager():
    from b200 import capi
    S, k, frames = 8, 96, 12
    scenes = [ts.scene(50 + s, frames, objects=20, k=k, crossings=2) for s in range(S)]
    batches = [[torch.from_numpy(np.stack([scenes[s][f][i] for s in range(S)])).cuda() for i in range(3)] for f in range(frames)]
    stamps = [torch.full((S,), f / 25.0, dtype=torch.float64, device="cuda") for f in range(frames)]
    zones = [capi.Zones(S), capi.Zones(S)]
    speeds = [capi.SpeedEstimator(S, min_samples=3), capi.SpeedEstimator(S, min_samples=3)]
    trackers = [capi.Tracker(S), capi.Tracker(S)]
    for z, e in zip(zones, speeds):
        for s in range(S):
            z.set(s, *zs.layout(s))
            e.set(s, _camera_h(s))
    static = [x.clone() for x in batches[0]] + [stamps[0].clone()]

    def step(trk, z, e, inp):
        ids, _, labels, boxes, _, counts = trk.update(*inp[:3], max_out=64)
        return z.update(ids, labels, boxes, counts, max_events=32) + e.update(ids, boxes, counts, timestamps=inp[3])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                       # warm-up outside the capture: one eager frame on both
        for t in (0, 1):
            step(trackers[t], zones[t], speeds[t], batches[0] + [stamps[0]])
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step(trackers[0], zones[0], speeds[0], static)
    for f in range(1, frames):
        for x, y in zip(static, batches[f] + [stamps[f]]):
            x.copy_(y)
        g.replay()
        want = step(trackers[1], zones[1], speeds[1], batches[f] + [stamps[f]])
        for a, b in zip(out, want):
            assert torch.equal(a, b) or (a.is_floating_point() and _same(a.cpu().numpy(), b.cpu().numpy())), f
    for s in range(S):
        a, b = speeds[0].export(s), speeds[1].export(s)
        assert all(_same(a[k_], b[k_]) for k_ in a if k_ != "samples")
        assert all(_same(x, y) for x, y in zip(a["samples"], b["samples"]))


def test_export_waits_for_the_object_only():
    from test_state_export_gpu import _equal, _exports_while_the_device_is_busy
    S = 4
    pair = Pair(S, min_samples=2)
    data = tracked(S, 3, seed=20)
    for ids, boxes, counts in data[:2]:
        pair.update(ids, boxes, counts, list(range(S)))
    got, after = _exports_while_the_device_is_busy(lambda: pair.dev.update(*data[2], list(range(S))),
                                                   lambda: [pair.dev.export(s) for s in range(S)])
    assert _equal(got, after)


def test_track_with_speed_equals_spec_on_the_returned_tracks():
    from b200 import capi
    from test_track_gpu import LOW, _model
    model = _model()
    rng = np.random.default_rng(5)
    base = [rng.integers(0, 256, (720, 1280, 3), dtype=np.uint8) for _ in range(3)]
    t_with, t_without = capi.Tracker(3, **LOW), capi.Tracker(3, **LOW)
    est = capi.SpeedEstimator(3, min_samples=2)
    spec = [sp.Stream(sp.params(min_samples=2)) for _ in range(3)]
    for s in range(3):
        est.set(s, _camera_h(s))
        spec[s].set(_camera_h(s))
    estimates = 0
    for call in range(4):
        streams = [0, 1, 0, 2]
        frames = [torch.from_numpy(np.roll(base[st], 24 * (call * 4 + i), axis=1)).cuda() for i, st in enumerate(streams)]
        stamps = [0.1 * (call * 4 + i) for i in range(4)] if call % 2 else None
        got = model.track(frames, t_with, streams=streams, speed=est, timestamps=stamps)
        plain = model.track(frames, t_without, streams=streams)
        for i, (st, d, e) in enumerate(zip(streams, got, plain)):
            assert all(torch.equal(d[k], e[k]) for k in e) and set(d) == set(e) | {"position", "velocity", "speed"}
            c = len(d["ids"])
            kin, _ = spec[st].update(d["ids"].cpu().numpy(), d["boxes"].cpu().numpy(), c, None if stamps is None else stamps[i])
            assert _same(d["position"].cpu().numpy(), kin[:c, :2]) and _same(d["velocity"].cpu().numpy(), kin[:c, 2:4])
            assert _same(d["speed"].cpu().numpy(), kin[:c, 4])
            estimates += int(np.isfinite(kin[:c, 4]).sum())
    for s in range(3):
        a, b = est.export(s), spec[s].export()
        assert all(_same(a[k], b[k]) for k in b if k != "samples")
    assert estimates > 0


def test_speed_rejections():
    from b200 import capi
    for bad in (dict(capacity=4097), dict(window=1), dict(window=65), dict(min_samples=31), dict(forget_after=-1), dict(anchor=9),
                dict(frame_rate=0.0)):
        with pytest.raises(RuntimeError):
            capi.SpeedEstimator(2, **bad)
    e = capi.SpeedEstimator(2)
    for H in (np.zeros((3, 3)), np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1.0]]), np.full((3, 3), np.inf)):
        with pytest.raises(ValueError):
            e.set(0, H)
    with pytest.raises(RuntimeError):                    # the C call's own check, past the Python one
        capi.check(capi.lib().lwdetr_speed_set(e._t, 0, np.zeros(9).ctypes.data_as(capi._vp)), "lwdetr_speed_set")
    with pytest.raises(ValueError):
        e.set(2, np.eye(3))
    ids = torch.ones(2, 4, dtype=torch.int32, device="cuda")
    boxes = torch.zeros(2, 4, 4, device="cuda")
    counts = torch.full((2,), 4, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        e.update(ids, boxes, counts, [0, 0])
    with pytest.raises(RuntimeError):
        e.update(ids, boxes, counts, [0, 2])
    big = torch.ones(1, 1025, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        e.update(big, torch.zeros(1, 1025, 4, device="cuda"), counts[:1])
    from test_track_gpu import _model
    model = _model()
    frames = [torch.zeros(64, 64, 3, dtype=torch.uint8, device="cuda")]
    with pytest.raises(RuntimeError):
        model.track(frames, capi.Tracker(1), speed=capi.SpeedEstimator(1), motion=capi.MotionEstimator(1))
