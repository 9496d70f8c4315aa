"""The exports of the device tracker and the camera-motion estimator wait for the object's own last launch and for nothing
else on the device: with about a second of unrelated work queued on another stream, Tracker.export / export_embeddings
and MotionEstimator.export return before that work ends, with the state a full device synchronise would show."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402

SLEEP_CYCLES = 2_000_000_000      # about a second at the H100's boost clock


def _exports_while_the_device_is_busy(launch, export):
    """launch() on the current stream, then a bounded spin kernel on a side stream; export() must return while it spins
    and equal export() after a full synchronise."""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(1000)                       # loads the spin kernel before the timed part
    torch.cuda.synchronize()
    launch()
    busy = torch.cuda.Event()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        busy.record()
    got = export()
    pending = not busy.query()
    torch.cuda.synchronize()
    assert pending, "the export waited for work on another stream"
    return got, export()


def _equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and np.array_equal(a, b)
    return a == b


@pytest.mark.parametrize("appearance", [False, True])
def test_tracker_export_waits_for_the_tracker_only(appearance):
    from b200 import capi
    S, k, D = 4, 64, 32
    frames = [ts.scene(70 + s, 2, objects=15, k=k) for s in range(S)]
    batch = [torch.from_numpy(np.stack([frames[s][f][i] for s in range(S)])).cuda() for f in range(2) for i in range(3)]
    tracker = capi.Tracker(S, embedding_dim=D) if appearance else capi.Tracker(S)
    emb = torch.randn(S, k, D, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) if appearance else None
    tracker.update(*batch[:3], embeddings=emb)

    def export():
        out = [tracker.export(s) for s in range(S)]
        return out + [tracker.export_embeddings(s) for s in range(S)] if appearance else out
    got, want = _exports_while_the_device_is_busy(lambda: tracker.update(*batch[3:], embeddings=emb), export)
    assert _equal(got, want)
    assert sum(len(recs) for recs, _ in want[:S]) > 0
    if appearance:
        assert any(has.any() for _, has in want[S:])


def test_estimator_export_waits_for_the_estimator_only():
    from b200 import capi
    S, h, w = 2, 360, 640
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (h + 8, w + 8, 3), dtype=np.uint8)
    est = capi.MotionEstimator(S, max_height=h, max_width=w)
    est.estimate([torch.from_numpy(base[s:s + h, :w].copy()).cuda() for s in range(S)])
    second = [torch.from_numpy(base[s + 2:s + 2 + h, 3:w + 3].copy()).cuda() for s in range(S)]
    got, want = _exports_while_the_device_is_busy(lambda: est.estimate(second), lambda: [est.export(s) for s in range(S)])
    assert _equal(got, want)
    assert all(st["valid"] and len(st["levels"]) > 1 and len(st["corners"]) > 0 and len(st["flow"]) > 0 for st in want)
