"""The per-object flow's specification (tools/flow_spec.py) on rendered sprites with cv2's Lucas-Kanade, and the tracker's
flow frames (track_spec.Stream.update_flow) on synthetic detection sequences."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import flow_spec as fs  # noqa: E402
import gmc_spec as gs  # noqa: E402
import track_spec as ts  # noqa: E402

cv2 = pytest.importorskip("cv2")


def _lk(a, b, pts, nlev, p):
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, p["iterations"], float(p["eps"]))
    kw = dict(winSize=(p["window"], p["window"]), maxLevel=nlev, criteria=crit, minEigThreshold=float(p["min_eig"]))
    q, s1, _ = cv2.calcOpticalFlowPyrLK(a, b, pts.reshape(-1, 1, 2), None, **kw)
    r, s2, _ = cv2.calcOpticalFlowPyrLK(b, a, q, None, **kw)
    return q.reshape(-1, 2), r.reshape(-1, 2), (s1.reshape(-1) == 1) & (s2.reshape(-1) == 1)


def _sprite_cases(seed, occluders, objects):
    """Per (frame, sprite) of a rendered scene with sprite 0 texture-less: (sprite, hidden, status, largest side error)."""
    p, g = fs.params(), gs.params()
    frames, boxes, hidden = fs.sprite_scene(seed, 6, objects=objects, occluders=occluders, flat=1)
    d = g["downscale"]
    nlev = gs.geometry(1080, 1920, g)[1]
    out = []
    for f in range(1, len(frames)):
        a, b = gs.level0(gs.grey_rgb(frames[f - 1]), d), gs.level0(gs.grey_rgb(frames[f]), d)
        for k in range(objects):
            mean = ts.measurement(boxes[f - 1, k].astype(np.float32))
            sd = fs.seeds(mean, p["grid"], d)
            fwd, bwd, ok = _lk(a, b, sd, nlev, p)
            st, _, _, _, z, _, _ = fs.measure(mean, sd, fwd, bwd, ok, a, b, p, d)
            err = np.abs(fs.box_of(z) - boxes[f, k]).max() if st == fs.OK else np.nan
            out.append((k, bool(hidden[f, k] or hidden[f - 1, k]), st, err))
    return out


@pytest.mark.parametrize("seed", [3, 4, 6])
def test_measurement_boxes_follow_rendered_sprites(seed):
    """Every textured sprite that nothing covers is measured (status OK) and its box is within 1.1 px of the truth on every
    side.  The 0.5 px asked for is not met: the worst sprites of these scenes are 0.54 / 0.96 / 0.48 px off (include/
    lwdetr_b200.h states it)."""
    cases = [c for c in _sprite_cases(seed, 0, 4) if c[0] != 0 and not c[1]]
    assert len(cases) >= 10
    assert all(st == fs.OK for _, _, st, _ in cases)
    errs = np.array([e for _, _, _, e in cases])
    print("seed %d: %d sprite frames, worst side error %.3f px, %.0f %% within 0.5 px" % (seed, len(errs), errs.max(), 100 * (errs <= 0.5).mean()))
    assert errs.max() <= 1.1


@pytest.mark.xfail(strict=True, reason="Median Flow can measure a texture-less or partly covered object from its outline and "
                   "give it a wrong box with status OK (include/lwdetr_b200.h); this test states the property that does not hold")
@pytest.mark.parametrize("seed", [3, 5])
def test_occluded_or_flat_sprites_fail_rather_than_mislead(seed):
    bad = [(k, st, e) for k, hidden, st, e in _sprite_cases(seed, 1, 4) if (k == 0 or hidden) and st == fs.OK and e > 1.1]
    print("seed %d: flat or covered sprites measured OK with a box more than 1.1 px off: %s" % (seed, bad))
    assert not bad


def test_statuses_and_medians():
    p = fs.params(min_points=3)
    rng = np.random.default_rng(0)
    img = (rng.random((200, 200)) * 255).astype(np.uint8)
    mean = np.array([100.0, 100.0, 1.0, 40.0])
    sd = fs.seeds(mean, 4, 2)
    assert sd.shape == (16, 2) and sd.dtype == np.float32
    # a pure translation of 2 level-0 px: dx = 4 frame px, s = 1
    fwd = (sd + np.float32(2.0)).astype(np.float32)
    st, dx, dy, s, z, fb, nc = fs.measure(mean, sd, fwd, sd.copy(), np.ones(16, bool), img, img, p, 2)
    assert st == fs.OK and dx == 4.0 and dy == 4.0 and s == 1.0 and np.array_equal(z, [104.0, 104.0, 1.0, 40.0])
    assert np.all(fb == 0)
    # nothing valid
    assert fs.measure(mean, sd, fwd, sd, np.zeros(16, bool), img, img, p, 2)[0] == fs.FEW_POINTS
    # large forward-backward error
    assert fs.measure(mean, sd, fwd, sd + np.float32(20), np.ones(16, bool), img, img, p, 2)[0] == fs.FB
    # a scale of 3 is outside [0.5, 2]
    c = sd.mean(0)
    st = fs.measure(mean, sd, ((sd - c) * 3 + c).astype(np.float32), sd, np.ones(16, bool), img, img, p, 2)[0]
    assert st == fs.SCALE
    # a zero-variance patch has NCC -1
    flat = np.full((200, 200), 7, np.uint8)
    assert fs.ncc(flat, img, (50.0, 50.0), (50.0, 50.0), 11) == -1.0
    assert fs.lower_median([3.0, 1.0, 2.0, 4.0]) == 2.0


def _object_boxes(frame, truth):
    return {int(o): frame[2][i] for i, o in enumerate(truth) if o >= 0}


@pytest.mark.parametrize("every", [2, 4])
def test_identities_survive_flow_frames(every):
    """True boxes as flow measurements: the flow frames keep every identity a detection on every frame keeps; an object
    without a box on a flow frame (occluded, missed) goes Lost and is refound at the next keyframe."""
    seq, _, truth = ts.scene(11, 120, objects=12, clutter=0, miss=0.02, occlusion=0.01, crossing=False, truth=True)
    p = ts.params()

    def run(n):
        st, owner, outs = ts.Stream(p), {}, []
        for f, (fr, g) in enumerate(zip(seq, truth)):
            if f % n == 0:
                o = st.update(*fr)
                for tid, _, _, _, idx in o:
                    owner[tid] = int(g[idx])
                outs.append(o)
                continue
            have = _object_boxes(fr, g)
            conf = [t for t in st.tracked if t.activated]
            meas = [(0, ts.measurement(have[owner[t.id]])) if owner.get(t.id) in have else (fs.FEW_POINTS, None) for t in conf]
            st.update_flow(meas)
            for t, (s_, _) in zip(conf, meas):
                assert (t.state == ts.LOST) == (s_ != 0)
        return outs                              # the keyframes' outputs
    every1 = ts.id_switches(run(1), truth)
    sw = ts.id_switches(run(every), truth[::every])
    print("identity switches: every frame %d, detect_every=%d %d" % (every1, every, sw))
    assert sw <= every1


def test_occluded_track_is_lost_then_refound():
    p = ts.params()
    st = ts.Stream(p)
    box = np.array([[100, 100, 180, 260]], np.float32)
    for _ in range(3):
        st.update(np.array([0.9], np.float32), np.array([0], np.int32), box)
    tid = st.tracked[0].id
    st.update_flow([(fs.FEW_POINTS, None)])
    assert not st.tracked and st.lost[0].id == tid and st.lost[0].state == ts.LOST
    out = st.update(np.array([0.9], np.float32), np.array([0], np.int32), box)
    assert [o[0] for o in out] == [tid]
