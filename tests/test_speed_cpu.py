"""The speed contract (include/lwdetr_b200.h, lwdetr_speed_*) as restated in tools/speed_spec.py: the calibration helper
capi.homography, accuracy on a synthetic road scene seen by a pinhole camera (exact up to fp32 box rounding without
noise, measured with noise, and through the ByteTrack specification), and the record lifecycle: forgetting, overflow,
reset, set, absent streams, bad clocks, the horizon, min_samples and the entry rule."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "lw-detr_b200"))

import speed_spec as sp  # noqa: E402
import track_spec as ts  # noqa: E402

# 1920 x 1080 frame: four image points of a 7 m x 40 m road rectangle
SRC = [(640.0, 1000.0), (1300.0, 1000.0), (1020.0, 420.0), (900.0, 420.0)]
DST = [(0.0, 0.0), (7.0, 0.0), (7.0, 40.0), (0.0, 40.0)]


def _homography():
    from b200 import capi
    return capi.homography


def test_homography_maps_its_points_and_matches_opencv():
    H = _homography()(SRC, DST)
    X, Y, ok = sp.project(H, np.array(SRC)[:, 0], np.array(SRC)[:, 1])
    assert ok.all()
    assert np.abs(np.stack([X, Y], 1) - np.array(DST)).max() < 1e-9
    cv2 = pytest.importorskip("cv2")
    ref = cv2.getPerspectiveTransform(np.float32(SRC), np.float32(DST))      # h8 = 1, whatever the sign of w
    assert abs(H[2, 2]) == 1.0
    assert np.allclose(H, H[2, 2] * ref, rtol=1e-9, atol=1e-12)


def test_homography_recovers_the_camera_and_normalises_w():
    cam = sp.camera()
    ground = np.array([(-5.0, 20.0, 0.0), (5.0, 20.0, 0.0), (5.0, 60.0, 0.0), (-5.0, 60.0, 0.0)])
    H = _homography()(sp.to_pixels(cam["P"], ground), ground[:, :2])
    assert np.allclose(H, cam["H"], rtol=1e-9, atol=1e-12)
    Hn = _homography()(SRC, [(0.0, 0.0), (7.0, 0.0), (7.0, -40.0), (0.0, -40.0)])   # any ground orientation
    cx, cy = np.mean(SRC, 0)
    assert Hn[2, 0] * cx + Hn[2, 1] * cy + Hn[2, 2] > 0


def test_homography_refuses_collinear_points():
    h = _homography()
    with pytest.raises(ValueError):
        h([(0, 0), (1, 1), (2, 2), (0, 5)], DST)
    with pytest.raises(ValueError):
        h(SRC, [(0, 0), (1, 0), (2, 0), (0, 5)])
    with pytest.raises(ValueError):
        h(SRC[:3], DST[:3])


def _jacobian_norm(H, x, y):
    """Frobenius norm of d(X, Y)/d(x, y) of the pixel -> ground map at (x, y)."""
    h = np.asarray(H).reshape(-1)
    a, b, w = h[0] * x + h[1] * y + h[2], h[3] * x + h[4] * y + h[5], h[6] * x + h[7] * y + h[8]
    J = np.array([[h[0] * w - a * h[6], h[1] * w - a * h[7]], [h[3] * w - b * h[6], h[4] * w - b * h[7]]]) / w ** 2
    return np.sqrt((J ** 2).sum())


def test_noise_free_speeds_within_the_fp32_rounding_bound():
    """Without noise the only error is the rounding of each box to fp32.  Every coordinate is below 2048 px in magnitude,
    so each edge moves by at most half an ulp there, eps = 2^-14 px, and so do the anchor's x = (x1 + x2) / 2 (exact in
    float64) and y = y2.  A pixel error of at most eps per coordinate moves sample i's ground point by at most
    |J_i|_F eps sqrt(2) (J_i the map's Jacobian there, to first order: 1 % slack covers the rest).  The fit is linear in
    the ground points with weights d_i / Stt (d_i = tau_i - mean tau), so the velocity, and with it the speed, moves by at
    most sum |d_i| |J_i|_F eps sqrt(2) / Stt.  On top: the fp32 rounding of the output (2^-24 relative) and float64
    rounding (1e-9 relative, far above it)."""
    boxes, vel, cam = sp.road_scene(1, objects=400)
    assert np.abs(boxes[..., [0, 2, 3]]).max() < 2048
    kin, n, s = sp.estimate_scene(boxes, cam["H"])
    true = np.hypot(*vel.T)
    eps = 2.0 ** -14
    ex = s.export()
    worst = 0.0
    for o, smp in enumerate(ex["samples"]):
        assert len(smp) == 30 and n[o] == 30
        tau = smp[:, 0] - smp[-1, 0]
        d = tau - tau.mean()
        J = np.array([_jacobian_norm(cam["H"], x, y) for x, y in smp[:, 1:]])
        bound = 1.01 * (np.abs(d) * J).sum() * eps * np.sqrt(2) / (d * d).sum() + (2.0 ** -24 + 1e-9) * true[o]
        err = abs(float(kin[o, 4]) - true[o])
        assert err <= bound, (o, err, bound)
        worst = max(worst, err / bound)
    assert worst > 0.01          # the bound is not vacuous: rounding shows


def test_identity_and_integer_pixels_give_the_exact_velocity():
    """H the identity and boxes on integer pixels moving whole pixels per frame: the ground points are exact, so float64
    rounding of tau (t = frame / 30) is the only error left."""
    rng = np.random.default_rng(4)
    n, frames = 50, 40
    x0, y0 = rng.integers(200, 1700, n), rng.integers(300, 900, n)
    kx, ky = rng.integers(-6, 7, n), rng.integers(-4, 5, n)
    f = np.arange(frames)[:, None]
    x, y = x0 + kx * f, y0 + ky * f
    boxes = np.stack([x - 20, y - 60, x + 20, y], -1).astype(np.float32)
    kin, samples, _ = sp.estimate_scene(boxes, np.eye(3))
    want = np.stack([kx, ky], 1) * 30.0
    got = kin[:, 2:4].astype(np.float64)
    moving = np.hypot(kx, ky) > 0
    assert (samples == 30).all()
    assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want) + 2.0 ** -24 * np.abs(want) + 1e-12)
    assert np.all(np.abs(kin[moving, 4] - np.hypot(*want[moving].T)) <= 2.0 ** -23 * np.hypot(*want[moving].T))


# Measured on road_scene(1, objects=400) at the defaults (window 30, min_samples 15, 30 fps): median and 95th percentile of
# |speed - truth| / truth.  supervision's endpoint estimator (|Y_first - Y_last| / (len / fps), ground y alone) on the same
# samples: 0.298 / 0.927 at sigma 1 and 0.299 / 0.949 at sigma 2 (random headings: y alone misses the rest of the motion).
NOISY = {1.0: (0.0019042, 0.0137652), 2.0: (0.0038311, 0.0282045)}


@pytest.mark.parametrize("sigma", [1.0, 2.0])
def test_noisy_speeds_match_the_recorded_errors(sigma):
    boxes, vel, cam = sp.road_scene(1, objects=400, sigma=sigma)
    kin, _, s = sp.estimate_scene(boxes, cam["H"])
    true = np.hypot(*vel.T)
    rel = np.abs(kin[:, 4] - true) / true
    med, p95 = NOISY[sigma]
    assert abs(np.median(rel) - med) <= 0.05 * med
    assert abs(np.percentile(rel, 95) - p95) <= 0.05 * p95
    ep = np.array([sp.endpoint_speed(r, cam["H"], 30.0) for r in s.export()["samples"]])
    assert np.median(np.abs(ep - true) / true) > 10 * med


def test_through_the_tracker_spec_the_speeds_stay_within_the_one_pixel_errors():
    """Noise-free scenes through track_spec.Stream (ByteTrack's Kalman boxes), then the speed spec: on tracks with a full
    window, the median and 95th percentile stay within those of 1 px of edge noise on the raw boxes."""
    rel = []
    for seed in range(12):
        boxes, vel, cam = sp.road_scene(100 + seed, objects=6, frames=60)
        trk = ts.Stream(ts.params())
        st = sp.Stream(sp.params())
        st.set(cam["H"])
        n = boxes.shape[1]
        for f in range(boxes.shape[0]):
            outs = trk.update(np.full(n, 0.9, np.float32), np.zeros(n, np.int32), boxes[f])
            ids, _, _, bx, ix, c = ts.outputs_array(outs, 16)
            kin, samples = st.update(ids, bx, c)
        for j in range(c):
            if ix[j] >= 0 and samples[j] == 30:
                true = np.hypot(*vel[ix[j]])
                rel.append(abs(kin[j, 4] - true) / true)
    assert len(rel) > 40
    assert np.median(rel) <= NOISY[1.0][0] and np.percentile(rel, 95) <= NOISY[1.0][1]


# ---------------------------------------------------------------------------------------------- lifecycle
def frame(tracks, max_out=None):
    """[(id, (x1, y1, x2, y2)), ...] -> (ids, boxes, count) padded as the tracker pads its outputs."""
    m = max(len(tracks), 1) if max_out is None else max_out
    ids = np.zeros(m, np.int32)
    boxes = np.zeros((m, 4), np.float32)
    for j, (i, b) in enumerate(tracks):
        ids[j], boxes[j] = i, b
    return ids, boxes, len(tracks)


def box(x, y):
    return (x - 10.0, y - 30.0, x + 10.0, y)


def test_forget_after_and_min_samples():
    s = sp.Stream(sp.params(forget_after=2, min_samples=3, window=4))
    for f in range(3):
        kin, n = s.update(*frame([(1, box(100 + 3 * f, 200))]))
    assert n[0] == 3 and np.isclose(kin[0, 2], 90.0) and kin[0, 3] == 0
    for f in range(3):
        s.update(*frame([]))
    assert s.export()["records"] == 0                  # absent for 3 > forget_after frames
    kin, n = s.update(*frame([(1, box(0, 0))]))
    assert n[0] == 1 and np.isnan(kin[0, 2:]).all()    # a new record: fewer than min_samples
    s2 = sp.Stream(sp.params(min_samples=2, window=3))
    for f in range(5):
        kin, n = s2.update(*frame([(7, box(10 * f, 500))]))
    assert n[0] == 3 and len(s2.export()["samples"][0]) == 3   # the ring keeps the last `window`


def test_capacity_overflow():
    s = sp.Stream(sp.params(capacity=2))
    kin, n = s.update(*frame([(1, box(10, 10)), (2, box(20, 20)), (3, box(30, 30))]))
    assert s.overflow == 1 and n.tolist() == [1, 1, 0]
    assert kin[2, 0] == 30 and np.isnan(kin[2, 2:]).all()     # position without a record
    assert s.export()["ids"].tolist() == [1, 2]


def test_reset_keeps_h_and_set_keeps_the_history():
    s = sp.Stream(sp.params(min_samples=2))
    for f in range(4):
        s.update(*frame([(1, box(100 + f, 100))]))
    H = np.diag([2.0, 2.0, 1.0])
    s.set(H)
    kin, n = s.update(*frame([(1, box(104, 100))]))
    assert n[0] == 5 and np.isclose(kin[0, 2], 60.0) and kin[0, 0] == 208   # all five samples, projected by the new H
    s.reset()
    e = s.export()
    assert (e["frame"], e["records"], e["clock_errors"], e["last_t"]) == (1, 0, 0, -np.inf)
    assert np.array_equal(e["homography"], H)


def test_absent_stream_does_not_advance_and_bad_clocks_are_counted():
    s = sp.Stream(sp.params(min_samples=2))
    s.update(*frame([(1, box(0, 0))]), t=1.0)
    s.update(*frame([(1, box(5, 0))]), t=1.0)           # not later
    s.update(*frame([(1, box(9, 0))]), t=np.nan)
    s.update(*frame([(1, box(7, 0))]), t=0.5)           # earlier
    kin, n = s.update(*frame([(1, box(10, 0))]), t=1.5)
    e = s.export()
    assert e["clock_errors"] == 3 and e["frame"] == 6 and e["last_t"] == 1.5
    assert n[0] == 2 and kin[0, 2] == 20.0
    assert [tuple(r) for r in e["samples"][0]] == [(1.0, 0.0, 0.0), (1.5, 10.0, 0.0)]


def test_points_beyond_the_horizon_are_nan():
    H = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, -0.01, 5.0]])     # w = 5 - y / 100: the horizon at y = 500
    s = sp.Stream(sp.params(min_samples=2))
    s.set(H)
    for f in range(3):
        kin, n = s.update(*frame([(1, box(100 + f, 400)), (2, box(100 + f, 500)), (3, box(100, 600 + f))]))
    assert np.isfinite(kin[0]).all() and n[0] == 3
    assert np.isnan(kin[1]).all() and np.isnan(kin[2]).all() and n[1] == n[2] == 0


def test_repeated_zero_and_non_finite_entries():
    s = sp.Stream(sp.params())
    ids, boxes, _ = frame([(4, box(1, 1)), (4, box(2, 2)), (0, box(3, 3)), (-1, box(4, 4)), (5, (np.nan, 0, 1, 1)), (6, box(6, 6))],
                          max_out=8)
    kin, n = s.update(ids, boxes, 7)
    assert n.tolist() == [1, 0, 0, 0, 0, 1, 0, 0]
    assert np.isfinite(kin[[0, 5], :2]).all() and np.isnan(kin[[1, 2, 3, 4, 6, 7]]).all()
    kin, n = s.update(ids, boxes, 1)                      # entries past the count are absent
    assert n.tolist() == [2, 0, 0, 0, 0, 0, 0, 0]


def test_parameter_and_homography_checks():
    for bad in (dict(capacity=0), dict(capacity=4097), dict(window=1), dict(window=65), dict(min_samples=1),
                dict(window=10, min_samples=11), dict(forget_after=-1), dict(anchor=9), dict(frame_rate=0.0),
                dict(frame_rate=np.inf)):
        with pytest.raises(ValueError):
            sp.params(**bad)
    for H in (np.zeros((3, 3)), np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1.0]]), np.full((3, 3), np.nan), np.eye(2)):
        with pytest.raises(ValueError):
            sp.check_homography(H)
