"""CPU tests of camera-motion compensation: the estimator's specification (tools/gmc_spec.py) against OpenCV for the grey,
downscale and pyramid rule, the corner response and the robust fit; the tracker specification's warp (tools/track_spec.py)
on moving-camera scenes."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gmc_spec as gs  # noqa: E402
import track_spec as ts  # noqa: E402

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("size", [(480, 640), (479, 637), (37, 53), (101, 77), (1080, 1920)])
def test_grey_downscale_and_pyramid_are_opencv_bit_for_bit(size):
    h, w = size
    rgb = gs.textured_frame(h * 7 + w, h, w)
    g = gs.grey_rgb(rgb)
    assert np.array_equal(g, cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))
    l0 = gs.level0(g, 2)
    if h % 2 == 0 and w % 2 == 0:
        assert np.array_equal(l0, cv2.resize(g, (w // 2, h // 2)))          # BoT-SORT's downscale
    lv = gs.pyramid(g, gs.params())
    for a, b in zip(lv, lv[1:]):
        assert np.array_equal(b, cv2.pyrDown(a))
    for d in (1, 3):
        l0 = gs.level0(g, d)
        assert l0.shape == (h // d, w // d)
        assert np.array_equal(gs.pyr_down(l0), cv2.pyrDown(l0))


def test_grey_weights_on_every_colour_channel_value():
    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)
    rgb[0, :256, 0] = np.arange(256)
    assert np.array_equal(gs.grey_rgb(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))


def test_corner_response_is_opencv_min_eigenvalue_up_to_its_scale():
    img = gs.level0(gs.grey_rgb(gs.textured_frame(3, 480, 640)), 2)
    R = gs.response(img) / (2 * 3060.0 ** 2)
    cv = cv2.cornerMinEigenVal(img, 3, 3).astype(np.float64)
    assert np.abs(R - cv).max() <= 1e-5 * cv.max()


def test_corner_rule_one_per_cell_spread_over_the_frame():
    p = gs.params()
    img = gs.level0(gs.grey_rgb(gs.textured_frame(4, 1080, 1920)), 2)
    pts = gs.corners(img, p)
    _, _, c, ncx, ncy = gs.geometry(1080, 1920, p)
    assert ncx * ncy <= p["max_points"] and (ncx - 1) * (ncy - 1) < p["max_points"] < (ncx + 1) * (ncy + 1)
    cells = (pts[:, 1] // c) * ncx + pts[:, 0] // c
    assert len(np.unique(cells)) == len(pts) and np.all(np.diff(cells) > 0)
    assert len(pts) > 0.9 * ncx * ncy
    flat = np.full_like(img, 77)
    assert len(gs.corners(flat, p)) == 0


def test_hypotheses_draw_distinct_pairs_in_range():
    for n in (2, 3, 10, 1000):
        i, j = gs.hypothesis_pairs(1024, n)
        assert i.min() >= 0 and j.min() >= 0 and i.max() < n and j.max() < n and np.all(i != j)
    i, j = gs.hypothesis_pairs(4096, 1000)
    assert len(set(zip(i.tolist(), j.tolist()))) > 4000


def test_refit_recovers_a_similarity_from_exact_pairs_with_30_percent_outliers():
    rng = np.random.default_rng(5)
    p = gs.params()
    for trial in range(5):
        truth = gs.similarity(rng.uniform(-3, 3), rng.uniform(0.95, 1.05), rng.uniform(-40, 40), rng.uniform(-40, 40), (960, 540))
        P = rng.uniform(0, [1920, 1080], (800, 2))
        Q = (np.c_[P, np.ones(len(P))] @ gs.matrix(truth).T)
        bad = rng.random(len(P)) < 0.3
        Q[bad] += rng.uniform(-200, 200, (bad.sum(), 2))
        m, status, inl, _ = gs.fit(P, Q, p)
        assert status == gs.OK
        assert np.abs(m - truth).max() < 1e-9, (trial, m - truth)
        assert inl >= (~bad).sum()


def test_fit_statuses():
    p = gs.params()
    P = np.random.default_rng(1).uniform(0, 500, (5, 2))
    m, st, _, _ = gs.fit(P, P, p)
    assert st == gs.FEW_POINTS and np.array_equal(m, [1, 0, 0, 0])
    P = np.random.default_rng(2).uniform(0, 500, (200, 2))
    Q = np.random.default_rng(3).uniform(0, 500, (200, 2))
    m, st, _, _ = gs.fit(P, Q, p)
    assert st == gs.FEW_INLIERS and np.array_equal(m, [1, 0, 0, 0])


def test_botsort_reference_recovers_a_known_motion():
    truth = gs.similarity(1.0, 1.02, 12.0, -7.0, (320, 240))
    prev, cur, _ = gs.moving_pair(11, 480, 640, truth, outlier_area=0.0)
    assert gs.corner_error(gs.botsort_gmc(prev, cur), truth, 480, 640) < 1.0


def _run(frames, motion=None, p=None):
    st = ts.Stream(p or ts.params())
    outs = [st.update(*fr, motion=None if motion is None else motion[f]) for f, fr in enumerate(frames)]
    return outs, st


def test_identity_motion_changes_nothing():
    frames = ts.scene(21, 120, objects=25, echo=0.05)
    ident = np.tile([1.0, 0.0, 0.0, 0.0], (len(frames), 1))
    a, sa = _run(frames)
    b, sb = _run(frames, ident)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for u, v in zip(x, y):
            assert u[0] == v[0] and u[4] == v[4] and np.array_equal(u[3], v[3])
    for u, v in zip(sa.export(), sb.export()):
        assert np.array_equal(u["mean"], v["mean"]) and np.array_equal(u["cov"], v["cov"])


def test_camera_scene_keeps_the_still_scene_and_its_draws():
    still = ts.scene(8, 40, k=64)
    moved, motion, truth = ts.scene(8, 40, k=64, camera=ts.CAMERA, truth=True)
    assert motion.shape == (40, 4) and np.array_equal(motion[0], [1, 0, 0, 0])
    assert np.abs(motion[1:, 2:]).max() > 5
    for s, m, g in zip(still, moved, truth):
        assert np.array_equal(s[0], m[0]) and np.array_equal(s[1], m[1]) and len(g) == 64
    again = ts.scene(8, 40, k=64, truth=True)[0]
    for s, a in zip(still, again):
        assert all(np.array_equal(x, y) for x, y in zip(s, a))


def test_xy_covariance_blocks_stay_equal_under_camera_motion():
    frames, motion, _ = ts.scene(31, 300, objects=25, camera=dict(ts.CAMERA, seed=3, rotate=0.5, zoom=0.01))
    st = ts.Stream(ts.params())
    n = 0
    for f, fr in enumerate(frames):
        st.update(*fr, motion=motion[f])
        for t in st.tracked + st.lost:
            assert t.P[0] == t.P[1] and t.C[0] == t.C[1] and t.V[0] == t.V[1]
            n += 1
    assert n > 3000


def test_warp_is_the_matrix_form_for_equal_xy_blocks():
    """The closed form equals applying the similarity to the 8 x 8 state and covariance (R = s Q on x, y and vx, vy; s on
    h and vh; 1 on the aspect) within rounding."""
    rng = np.random.default_rng(2)
    t = ts.Track()
    t.p, t.v = rng.uniform(1, 100, 4), rng.normal(0, 2, 4)
    P, C, V = rng.uniform(1, 5, 4), rng.uniform(0, 1, 4), rng.uniform(1, 5, 4)
    P[1], C[1], V[1] = P[0], C[0], V[0]
    t.P, t.C, t.V = P.copy(), C.copy(), V.copy()
    m = gs.similarity(2.0, 1.03, 5.0, -3.0)
    a, b = m[0], m[1]
    s = np.hypot(a, b)
    A4 = np.zeros((4, 4))
    A4[:2, :2] = [[a, -b], [b, a]]
    A4[2, 2], A4[3, 3] = 1.0, s
    A = np.kron(np.eye(2), A4)
    cov = np.block([[np.diag(P), np.diag(C)], [np.diag(C), np.diag(V)]])
    mean = A @ np.r_[t.p, t.v] + np.r_[m[2], m[3], 0, 0, 0, 0, 0, 0]
    cov2 = A @ cov @ A.T
    ts.warp(t, m)
    assert np.allclose(np.r_[t.p, t.v], mean, rtol=1e-12, atol=1e-9)
    assert np.allclose(np.block([[np.diag(t.P), np.diag(t.C)], [np.diag(t.C), np.diag(t.V)]]), cov2, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_true_motion_removes_the_id_switches_the_camera_causes(seed):
    still, _, g = ts.scene(seed, 300, objects=20, truth=True)
    cam, motion, gc = ts.scene(seed, 300, objects=20, camera=ts.CAMERA, truth=True)
    n_still = ts.id_switches(_run(still)[0], g)
    n_cam = ts.id_switches(_run(cam)[0], gc)
    n_comp = ts.id_switches(_run(cam, motion)[0], gc)
    print("seed %d: id switches still %d, moving camera %d, moving camera with its motion %d" % (seed, n_still, n_cam, n_comp))
    assert n_cam > n_still + 20
    assert n_comp <= n_still
