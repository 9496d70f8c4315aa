"""GPU tests of line crossings and zone occupancy: the kernel (csrc/zones.cu, lwdetr_zones_update) bit for bit against its
specification (tools/zone_spec.py) on device-tracker outputs for 1, 32 and 256 streams: inside masks, occupancy, events in
order and every export field, with changing stream subsets, geometry at the limits, set and reset mid-sequence; one CUDA
graph of Tracker.update + Zones.update replayed; an export that waits for the object's own work only; LWDETR.track(zones=)
against the specification run on the tracks it returned."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402
import zone_spec as zs  # noqa: E402


class Pair:
    """A device zones object and one specification stream per stream id, driven together."""

    def __init__(self, num_streams, **params):
        from b200 import capi
        self.dev = capi.Zones(num_streams, **params)
        self.spec = [zs.Stream(zs.params(**params)) for _ in range(num_streams)]
        self.events = 0

    def set(self, s, lines, polygons):
        self.dev.set(s, lines, polygons)
        self.spec[s].set(lines, polygons)

    def reset(self, streams):
        self.dev.reset(streams)
        for s in streams:
            self.spec[s].reset()

    def update(self, ids, labels, boxes, counts, streams, max_events=64):
        got = self.dev.update(ids, labels, boxes, counts, streams, max_events=max_events)
        self.check(got, ids, labels, boxes, counts, streams, max_events)

    def check(self, got, ids, labels, boxes, counts, streams, max_events):
        inside, occ, ev, ec = [t.cpu().numpy() for t in got]
        ids, labels, boxes, counts = [t.cpu().numpy() for t in (ids, labels, boxes, counts)]
        for b, s in enumerate(streams):
            w_in, w_occ, w_ev = self.spec[s].update(ids[b], labels[b], boxes[b], counts[b])
            rows, n = zs.events_array(w_ev, max_events)
            assert np.array_equal(inside[b].view(np.uint32), w_in), (s, inside[b].view(np.uint32), w_in)
            assert np.array_equal(occ[b], w_occ), s
            assert ec[b] == n, (s, ec[b], n)
            assert np.array_equal(ev[b], rows), (s, ev[b][:n], rows[:n])
            self.events += n

    def compare_exports(self, streams=None):
        for s in range(len(self.spec)) if streams is None else streams:
            got, want = self.dev.export(s), self.spec[s].export()
            assert got.keys() == want.keys()
            for k in want:
                g, w = np.asarray(got[k]), np.asarray(want[k])
                assert g.shape == w.shape and np.array_equal(g, w), (s, k, g, w)


def tracked(S, frames, seed=0, objects=25, max_out=64):
    """Device-tracker outputs over seeded scenes, one per stream: a list per frame of (ids, labels, boxes, counts) [S, ...]."""
    from b200 import capi
    k = 96
    scenes = [ts.scene(seed + s, frames, objects=objects, k=k, crossings=3) for s in range(S)]
    trk = capi.Tracker(S)
    out = []
    for f in range(frames):
        sc, lab, bx = (torch.from_numpy(np.stack([scenes[s][f][i] for s in range(S)])).cuda() for i in range(3))
        ids, _, labels, boxes, _, counts = trk.update(sc, lab, bx, max_out=max_out)
        out.append((ids, labels, boxes, counts))
    return out


@pytest.mark.parametrize("S,frames", [(1, 60), (32, 24), (256, 8)])
def test_kernel_equals_spec_with_subsets_set_and_reset(S, frames):
    rng = np.random.default_rng(S)
    pair = Pair(S, forget_after=4, capacity=40, num_classes=2)
    for s in range(S):
        pair.set(s, *zs.layout(s, lines=4, polygons=8, vertices=16))
    for f, (ids, labels, boxes, counts) in enumerate(tracked(S, frames, seed=100)):
        rows = np.sort(rng.choice(S, size=max(1, int(rng.integers(S // 2, S + 1))), replace=False)) if S > 1 and f % 3 else np.arange(S)
        rng.shuffle(rows)
        idx = torch.from_numpy(rows).cuda()
        pair.update(ids[idx], labels[idx], boxes[idx], counts[idx], rows.tolist())
        if f == frames // 2:
            pair.reset([int(x) for x in rows[: max(1, len(rows) // 4)]])
            pair.set(int(rows[-1]), *zs.layout(1000 + f, lines=3, polygons=5, vertices=7))
    pair.compare_exports()
    assert pair.events > 10 * S


def test_geometry_at_the_limits_and_truncated_events():
    pair = Pair(2, forget_after=3)
    lines, _ = zs.layout(7, lines=32, polygons=0)
    polys = [zs.star(960 + 300 * np.cos(a), 540 + 300 * np.sin(a), 250, 90, 32) for a in np.linspace(0, 6, 32)]   # 64 vertices
    assert sum(len(p) for p in polys) == 2048
    for s in range(2):
        pair.set(s, lines, polys)
    for ids, labels, boxes, counts in tracked(2, 30, seed=7, objects=40):
        pair.update(ids, labels, boxes, counts, [0, 1], max_events=8)
    pair.compare_exports()
    assert pair.events > 100


def test_overflow_duplicates_and_absent_entries():
    pair = Pair(1, capacity=5, num_classes=1)
    pair.set(0, [(0.0, 500.0, 1920.0, 520.0)], [[(0, 0), (1920, 0), (1920, 540), (0, 540)]])
    rng = np.random.default_rng(3)
    for f in range(20):
        n = 12
        ids = rng.integers(1, 9, n).astype(np.int32)            # repeats, and more ids than records
        ids[rng.random(n) < 0.2] = int(rng.integers(-2, 1))
        cy = rng.uniform(300, 800, n)
        boxes = np.stack([rng.uniform(0, 1800, n), cy - 40, rng.uniform(0, 1800, n) + 100, cy + 40], 1).astype(np.float32)
        boxes[rng.random(n) < 0.1, 2] = np.nan
        labels = rng.integers(-1, 3, n).astype(np.int32)
        t = [torch.from_numpy(x[None]).cuda() for x in (ids, labels, boxes)]
        pair.update(*t, torch.tensor([int(rng.integers(0, n + 3))], dtype=torch.int32, device="cuda"), [0], max_events=4)
    pair.compare_exports()
    assert pair.dev.export(0)["overflow"] > 0


def test_cuda_graph_of_track_and_zones_equals_eager():
    from b200 import capi
    S, k, frames = 8, 96, 12
    scenes = [ts.scene(50 + s, frames, objects=20, k=k, crossings=2) for s in range(S)]
    batches = [[torch.from_numpy(np.stack([scenes[s][f][i] for s in range(S)])).cuda() for i in range(3)] for f in range(frames)]
    geo = [zs.layout(s) for s in range(S)]
    zones = [capi.Zones(S), capi.Zones(S)]
    trackers = [capi.Tracker(S), capi.Tracker(S)]
    for z in zones:
        for s in range(S):
            z.set(s, *geo[s])
    static = [x.clone() for x in batches[0]]

    def step(trk, z, inp):
        ids, _, labels, boxes, _, counts = trk.update(*inp, max_out=64)
        return z.update(ids, labels, boxes, counts, max_events=32)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                       # warm-up outside the capture: one eager frame on both
        for t in (0, 1):
            step(trackers[t], zones[t], batches[0])
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step(trackers[0], zones[0], static)
    for f in range(1, frames):
        for x, y in zip(static, batches[f]):
            x.copy_(y)
        g.replay()
        want = step(trackers[1], zones[1], batches[f])
        for a, b in zip(out, want):
            assert torch.equal(a, b), f
    for s in range(S):
        a, b = zones[0].export(s), zones[1].export(s)
        assert all(np.array_equal(a[k_], b[k_]) for k_ in a)


def test_export_waits_for_the_object_only():
    from test_state_export_gpu import _equal, _exports_while_the_device_is_busy
    S = 4
    pair = Pair(S)
    for s in range(S):
        pair.set(s, *zs.layout(s))
    data = tracked(S, 3, seed=20)
    for ids, labels, boxes, counts in data[:2]:
        pair.update(ids, labels, boxes, counts, list(range(S)))
    got, after = _exports_while_the_device_is_busy(lambda: pair.dev.update(*data[2], list(range(S))),
                                                   lambda: [pair.dev.export(s) for s in range(S)])
    assert _equal(got, after)


def test_track_with_zones_equals_spec_on_the_returned_tracks():
    from b200 import capi
    from test_track_gpu import LOW, _model
    model = _model()
    rng = np.random.default_rng(5)
    base = [rng.integers(0, 256, (720, 1280, 3), dtype=np.uint8) for _ in range(3)]
    tracker, z = capi.Tracker(3, **LOW), capi.Zones(3, num_classes=model.cfg.num_classes)
    spec = [zs.Stream(zs.params(num_classes=model.cfg.num_classes)) for _ in range(3)]
    for s in range(3):
        geo = zs.layout(40 + s, size=(720, 1280), lines=6, polygons=8, vertices=12)
        z.set(s, *geo)
        spec[s].set(*geo)
    n_events = 0
    for call in range(4):
        streams = [0, 1, 0, 2]
        frames = [torch.from_numpy(np.roll(base[st], 24 * (call * 4 + i), axis=1)).cuda() for i, st in enumerate(streams)]
        got = model.track(frames, tracker, streams=streams, zones=z)
        for st, d in zip(streams, got):
            c = len(d["ids"])
            inside, occ, ev = spec[st].update(d["ids"].cpu().numpy(), d["labels"].cpu().numpy(), d["boxes"].cpu().numpy(), c)
            assert np.array_equal(d["inside"].cpu().numpy(), inside[:c].astype(np.int64))
            assert np.array_equal(d["occupancy"].cpu().numpy(), occ)
            assert np.array_equal(d["events"].cpu().numpy(), np.array(ev[:1024], np.int32).reshape(-1, 5))   # max_events
            n_events += len(ev)
    for s in range(3):
        got, want = z.export(s), spec[s].export()
        assert all(np.array_equal(got[k], want[k]) for k in want)
    assert n_events > 0


def test_zones_rejections():
    from b200 import capi
    with pytest.raises(RuntimeError):
        capi.Zones(2, capacity=4097)
    with pytest.raises(RuntimeError):
        capi.Zones(2, line_anchors=0)
    z = capi.Zones(2)
    ids = torch.ones(2, 4, dtype=torch.int32, device="cuda")
    boxes = torch.zeros(2, 4, 4, device="cuda")
    counts = torch.full((2,), 4, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        z.update(ids, ids, boxes, counts, [0, 0])
    with pytest.raises(RuntimeError):
        z.update(ids, ids, boxes, counts, [0, 2])
    big = torch.ones(1, 1025, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        z.update(big, big, torch.zeros(1, 1025, 4, device="cuda"), counts[:1])
