"""The line-crossing and zone contract (include/lwdetr_b200.h, lwdetr_zones_*) as restated in tools/zone_spec.py: crossing
directions, undecided frames, first sightings, lost and forgotten tracks, the even-odd rule on awkward polygons, counters,
truncation and overflow, and the geometry checks of capi.Zones.set, which run before any device call.  The line counts are
also checked against crossings counted directly from the true object paths of track_spec.scene."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import track_spec as ts  # noqa: E402
import zone_spec as zs  # noqa: E402


def frame(tracks, max_out=None):
    """[(id, label, (x1, y1, x2, y2)), ...] -> (ids, labels, boxes, count) padded as the tracker pads its outputs."""
    m = max(len(tracks), 1) if max_out is None else max_out
    ids = np.zeros(m, np.int32)
    labels = np.full(m, -1, np.int32)
    boxes = np.zeros((m, 4), np.float32)
    for j, (i, l, b) in enumerate(tracks):
        ids[j], labels[j], boxes[j] = i, l, b
    return ids, labels, boxes, len(tracks)


def box_at(cx, cy, w=10.0, h=10.0):
    return (cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2)


def stream(lines=(), polygons=(), **kw):
    s = zs.Stream(zs.params(**kw))
    s.set(lines, polygons)
    return s


def run(s, path, tid=1, label=0):
    """One track along the centres `path` (None: absent that frame); all events."""
    ev = []
    for c in path:
        ev += s.update(*frame([] if c is None else [(tid, label, box_at(*c))]))[2]
    return ev


LINE = (0.0, 100.0, 200.0, 100.0)          # left to right at y = 100


def test_both_directions_and_swapped_endpoints():
    s = stream([LINE])
    ev = run(s, [(100, 50), (100, 80), (100, 150), (100, 60)])
    assert ev == [(1, zs.LINE_IN, 0, 0, 0), (1, zs.LINE_OUT, 0, 0, 0)]      # downward is "in" for a line drawn left to right
    assert s.export()["line_counts"][0, 0].tolist() == [1, 1]
    s = stream([(200.0, 100.0, 0.0, 100.0)])
    assert [e[1] for e in run(s, [(100, 50), (100, 150)])] == [zs.LINE_OUT]


def test_straddling_and_outside_the_segment_do_not_count():
    s = stream([LINE])
    # above; straddling the line (corners on both sides); below but past either end of the segment: never decided below
    ev = run(s, [(100, 50), (100, 100), (250, 150), (100, 60), (-30, 150), (2, 150)])
    assert ev == []
    s = stream([LINE])
    ev = run(s, [(100, 50), (100, 100), (100, 150)])
    assert [e[1] for e in ev] == [zs.LINE_IN]                 # an undecided frame keeps the side
    assert zs.line_sides(np.array([box_at(196, 150)], np.float32), LINE, zs.CORNERS).tolist() == [0]   # x2 = 201 > 200
    assert zs.line_sides(np.array([box_at(195, 150)], np.float32), LINE, zs.CORNERS).tolist() == [1]   # x2 = 200: t = L2


def test_first_sighting_does_not_count():
    s = stream([LINE])
    assert run(s, [(100, 150)]) == []
    assert s.export()["sides"].tolist() == [[1]]
    assert s.export()["line_counts"].sum() == 0


def test_lost_then_refound_on_the_other_side_counts_once():
    s = stream([LINE], forget_after=30)
    ev = run(s, [(100, 50)] + [None] * 30 + [(100, 150), (100, 160)])
    assert ev == [(1, zs.LINE_IN, 0, 0, 0)]


def test_forgotten_then_seen_again_starts_fresh_and_forget_has_the_dwell():
    zone = [(0, 0), (200, 0), (200, 200), (0, 200)]
    s = stream([LINE], [zone], forget_after=5)
    # bottom-centre anchor: box_at(100, 50) has it at y = 55, inside
    ev = run(s, [(100, 50), (100, 50), (100, 50)] + [None] * 5)
    assert ev == [(1, zs.ZONE_ENTER, 0, 0, 0)]
    assert len(s.export()["ids"]) == 1
    ev = s.update(*frame([]))[2]                            # frame 9: 9 - 3 > 5
    assert ev == [(1, zs.ZONE_FORGET, 0, 0, 3 - 1)]
    assert len(s.export()["ids"]) == 0
    ev = run(s, [(100, 150)])                               # the same id again: a first sighting, a new entry
    assert ev == [(1, zs.ZONE_ENTER, 0, 0, 0)]
    assert s.export()["entries"][0, 0] == 2


def test_exit_dwell_and_occupancy():
    zone = [(0, 0), (200, 0), (200, 200), (0, 200)]
    s = stream([], [zone])
    out = [s.update(*frame([(1, 2, box_at(100, 50)), (2, 2, box_at(300, 50))])) for _ in range(4)]
    assert out[0][1][0] == 1 and out[0][0][:2].tolist() == [1, 0]
    inside, occ, ev = s.update(*frame([(1, 2, box_at(300, 50))]))
    assert ev == [(1, zs.ZONE_EXIT, 0, 2, 5 - 1)] and occ[0] == 0 and inside[0] == 0


def test_even_odd_on_awkward_polygons():
    square = np.array([(0, 0), (4, 0), (4, 4), (0, 4)], np.float64)
    # the half-open rule: bottom (smaller y) and left edges in, top and right edges out, the (0, 0) vertex in
    pts = [(2, 0), (2, 4), (0, 2), (4, 2), (0, 0), (4, 4), (2, 2), (5, 2)]
    got = zs.inside_polygon([p[0] for p in pts], [p[1] for p in pts], square).tolist()
    assert got == [True, False, True, False, True, False, True, False]
    diamond = np.array([(2, 0), (4, 2), (2, 4), (0, 2)], np.float64)       # the row y = 2 runs through two vertices
    assert zs.inside_polygon([1, 3, 5, -1], [2, 2, 2, 2], diamond).tolist() == [True, True, False, False]
    # concave; (3, 2) lies on the notch's horizontal edge, which has the inside below it: out, like the square's top edge
    notch = np.array([(0, 0), (6, 0), (6, 6), (4, 6), (4, 2), (2, 2), (2, 6), (0, 6)], np.float64)
    assert zs.inside_polygon([1, 3, 5, 3, 3], [4, 4, 4, 1, 2], notch).tolist() == [True, False, True, True, False]
    bowtie = np.array([(0, 0), (4, 4), (4, 0), (0, 4)], np.float64)        # self-intersecting
    assert zs.inside_polygon([0.5, 3.5, 2, 2], [2, 2, 0.5, 3.5], bowtie).tolist() == [True, True, False, False]
    pentagram = zs.star(0, 0, 10, 10, 5)                            # a star drawn with crossing edges: the centre is out
    order = np.array([0, 4, 8, 2, 6]) % 10
    assert zs.inside_polygon([0, 0], [0, 9.9], pentagram[order]).tolist() == [False, False]


def test_per_class_and_other_counters():
    s = stream([LINE], [[(0, 0), (200, 0), (200, 300), (0, 300)]], num_classes=3)
    for tid, lab in [(1, 0), (2, 2), (3, -1), (4, 7)]:
        run(s, [(100, 50), (100, 150)], tid=tid, label=lab)
    e = s.export()
    assert e["line_counts"][0, :, 0].tolist() == [1, 0, 1, 2] and e["line_counts"][0, :, 1].sum() == 0
    assert e["entries"][0].tolist() == [1, 0, 1, 2]


def test_truncation_keeps_the_true_count_and_overflow_is_counted():
    s = stream([LINE, (0.0, 120.0, 200.0, 120.0)], capacity=3)
    tracks = [(i + 1, 0, box_at(20 + 30 * i, 50)) for i in range(5)]
    inside, occ, ev = s.update(*frame(tracks))
    assert ev == [] and s.export()["overflow"] == 2 and len(s.export()["ids"]) == 3
    ev = s.update(*frame([(i, l, box_at((b[0] + b[2]) / 2, 150)) for i, l, b in tracks]))[2]
    assert len(ev) == 6                                    # 3 recorded tracks x 2 lines; the other 2 stay unrecorded
    rows, n = zs.events_array(ev, 4)
    assert n == 6 and rows.tolist() == [list(e) for e in ev[:4]]
    rows, n = zs.events_array(ev, 8)
    assert n == 6 and not rows[6:].any()
    assert s.export()["overflow"] == 4


def test_repeated_id_later_entries_are_ignored():
    zone = [(0, 0), (200, 0), (200, 200), (0, 200)]
    s = stream([], [zone])
    inside, occ, ev = s.update(*frame([(5, 0, box_at(300, 50)), (5, 1, box_at(100, 50)), (0, 0, box_at(100, 50))]))
    assert inside.tolist() == [0, 0, 0] and occ[0] == 0 and ev == []


def test_absent_entries_past_the_count_and_non_finite():
    zone = [(0, 0), (200, 0), (200, 200), (0, 200)]
    s = stream([], [zone])
    ids, labels, boxes, _ = frame([(1, 0, box_at(100, 50)), (2, 0, (np.nan, 0, 10, 10)), (3, 0, box_at(100, 50))])
    inside, occ, ev = s.update(ids, labels, boxes, 1)
    assert inside.tolist() == [1, 0, 0] and occ[0] == 1 and [e[0] for e in ev] == [1]
    inside, occ, ev = s.update(ids, labels, boxes, 3)
    assert inside.tolist() == [1, 0, 1] and [e[0] for e in ev] == [3]


def test_reset_and_set():
    s = stream([LINE])
    run(s, [(100, 50), (100, 150)])
    s.set([LINE], [])
    e = s.export()
    assert e["frame"] == 3 and len(e["ids"]) == 0 and e["line_counts"].sum() == 0
    s.reset()
    assert s.export()["frame"] == 1 and len(s.lines) == 1


def test_invariant_entries_minus_exits_minus_forgets_is_records_inside():
    lines, polys = zs.layout(3, lines=4, polygons=8, vertices=16)
    s = stream(lines, polys, forget_after=10, capacity=40)
    trk = ts.Stream(ts.params())
    enter = leave = 0
    for sc, lab, bx in ts.scene(5, 120, objects=25, k=None):
        ids, _, labels, boxes, _, n = ts.outputs_array(trk.update(sc, lab, bx), 64)
        _, _, ev = s.update(ids, labels, boxes, n)
        enter += sum(e[1] == zs.ZONE_ENTER for e in ev)
        leave += sum(e[1] in (zs.ZONE_EXIT, zs.ZONE_FORGET) for e in ev)
        e = s.export()
        assert enter - leave == sum(bin(int(m)).count("1") for m in e["inside"])
        assert enter == e["entries"].sum()
    assert enter > 20 and leave > 10


@pytest.mark.parametrize("line", [(-1e4, 540.0, 1e4, 540.0), (960.0, -1e4, 960.0, 1e4), (-1e4, -1e4 * 0.5 + 200, 1e4, 1e4 * 0.5 + 200)])
def test_line_counts_equal_crossings_of_the_true_paths(line):
    """The objects' own detections with their true identities as tracks: the spec's counts on the centre anchor equal the
    sign changes of the centre's side, counted directly between consecutive sightings of each object."""
    frames, _, truth = ts.scene(11, 150, objects=30, crossings=6, truth=True)
    s = stream([line], forget_after=10 ** 6, line_anchors=1 << zs.CENTER)
    ax, ay, bx, by = line
    last, want = {}, np.zeros(2, np.int64)
    for (sc, lab, bx_), g in zip(frames, truth):
        keep = g >= 0
        tracks = [(int(o) + 1, int(l), b) for o, l, b in zip(g[keep], lab[keep], bx_[keep])]
        s.update(*frame(tracks))
        for tid, _, b in tracks:
            cx, cy = (np.float64(b[0]) + np.float64(b[2])) * 0.5, (np.float64(b[1]) + np.float64(b[3])) * 0.5
            side = np.sign((bx - ax) * (cy - ay) - (by - ay) * (cx - ax))
            if side != 0:
                if last.get(tid, side) != side:
                    want[0 if side > 0 else 1] += 1
                last[tid] = side
    got = s.export()["line_counts"][0].sum(0)
    assert got.tolist() == want.tolist() and want.sum() > 0


def test_geometry_checks_before_any_device_call():
    from b200 import capi
    z = object.__new__(capi.Zones)            # no device object: set() must refuse before it reaches one
    z.num_streams, z._t = 2, None
    bad = [
        dict(lines=[LINE] * 33), dict(lines=[(1, 1, 1, 1)]), dict(lines=[(0, 0, np.inf, 1)]), dict(lines=[(0, 0, 1)]),
        dict(polygons=[[(0, 0), (1, 1)]]), dict(polygons=[[(0, 0), (1, 1), (np.nan, 0)]]),
        dict(polygons=[zs.regular_polygon(0, 0, 1, 257)]), dict(polygons=[zs.regular_polygon(0, 0, 1, 3)] * 33),
        dict(polygons=[zs.regular_polygon(0, 0, 1, 256)] * 8 + [zs.regular_polygon(0, 0, 1, 3)]),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            capi.Zones.set(z, 0, **kw)
        with pytest.raises(ValueError):
            zs.geometry(**kw)
    with pytest.raises(ValueError):
        capi.Zones.set(z, 2, lines=[LINE])
    ln, sizes, verts = capi.zone_geometry([LINE] * 32, [zs.regular_polygon(0, 0, 1, 64)] * 32)
    assert ln.shape == (32, 4) and sizes.sum() == 2048 and verts.shape == (2048, 2)
