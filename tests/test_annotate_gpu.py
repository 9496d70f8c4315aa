"""GPU tests of drawing into frames (csrc/annotate.cu, lwdetr_annotate / _nv12) bit for bit against tools/annotate_spec.py,
on every byte of every surface: the frames sit inside larger buffers with odd pitches, so the pitch padding and the bytes
around each frame must come back unchanged.  RGB and NV12 in all four colorspaces, odd and mixed sizes, B = 1, 32 and 256,
k = 1024, counts of 0, boxes partly or wholly outside, options at their limits, zones at their limits, privacy blocks cut by
the frame edge; one CUDA graph of Tracker.update + Zones.update + annotate replayed; LWDETR.track(annotate=) against
Annotator.draw."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import annotate_spec as an  # noqa: E402
import zone_spec as zs  # noqa: E402

NAMES = ["person", "bicycle", "car", "Mot\x7forbike", "a-very-long-class-name-of-31-ch", ""]


class Surfaces:
    """B frames, each inside a larger random buffer (rows above and below, bytes left and right, odd pitches)."""

    def __init__(self, sizes, nv12, rng, dev="cuda"):
        self.nv12, self.sizes, self.bufs, self.frames, self.where = nv12, sizes, [], [], []
        for h, w in sizes:
            if nv12:
                ch, cw = (h + 1) // 2, (w + 1) // 2
                lo, co = int(rng.integers(0, 5)), 2 * int(rng.integers(0, 3))
                lb = torch.from_numpy(rng.integers(0, 256, (h + 2, w + lo + int(rng.integers(1, 8))), dtype=np.uint8)).to(dev)
                cb = torch.from_numpy(rng.integers(0, 256, (ch + 2, 2 * cw + co + int(rng.integers(1, 8))), dtype=np.uint8)).to(dev)
                self.bufs.append((lb, cb))
                self.frames.append((lb[1:1 + h, lo:lo + w], cb[1:1 + ch, co:co + 2 * cw]))
                self.where.append((lo, co))
            else:
                off = int(rng.integers(0, 7))
                buf = torch.from_numpy(rng.integers(0, 256, (h + 2, 3 * w + off + int(rng.integers(1, 9))), dtype=np.uint8)).to(dev)
                self.bufs.append(buf)
                self.frames.append(torch.as_strided(buf, (h, w, 3), (buf.stride(0), 3, 1), buf.stride(0) + off))
                self.where.append(off)

    def host(self):
        return [tuple(t.cpu().numpy() for t in b) if self.nv12 else b.cpu().numpy() for b in self.bufs]

    def spec_draw(self, bufs, b, a, cs, **entries):
        """The specification on frame b of host copies `bufs` (in place)."""
        h, w = self.sizes[b]
        if self.nv12:
            lb, cb = bufs[b]
            lo, co = self.where[b]
            ch, cw = (h + 1) // 2, (w + 1) // 2
            luma, chroma = lb[1:1 + h, lo:lo + w].copy(), cb[1:1 + ch, co:co + 2 * cw].copy()
            a.draw_nv12(luma, chroma, cs, **entries)
            lb[1:1 + h, lo:lo + w] = luma
            cb[1:1 + ch, co:co + 2 * cw] = chroma
        else:
            off = self.where[b]
            img = bufs[b][1:1 + h, off:off + 3 * w].reshape(h, w, 3).copy()
            a.draw_rgb(img, **entries)
            bufs[b][1:1 + h, off:off + 3 * w] = img.reshape(h, 3 * w)


def entries(rng, sizes, k, nc, with_ids=True):
    B = len(sizes)
    hw = np.array(sizes, np.float32)
    c = rng.uniform(-0.2, 1.2, (B, k, 2)) * hw[:, None, ::-1]
    wh = rng.uniform(0.02, 0.5, (B, k, 2)) * hw[:, None, ::-1]
    boxes = np.concatenate([c - wh / 2, c + wh / 2], -1).astype(np.float32)
    boxes[rng.random((B, k)) < 0.03] = np.nan
    boxes[rng.random((B, k)) < 0.03, 2] = -5.0                          # empty
    scores = rng.uniform(0, 1, (B, k)).astype(np.float32)
    labels = rng.integers(-1, nc + 2, (B, k)).astype(np.int32)
    ids = rng.integers(1, 5000, (B, k)).astype(np.int32) if with_ids else None
    counts = rng.integers(0, k + 1, B).astype(np.int32)
    counts[0] = 0 if B > 1 else counts[0]
    return scores, labels, boxes, ids, counts


def check(sizes, nv12, cs, k=40, nc=6, seed=0, with_ids=True, zones=False, threshold=0.3, privacy=(1, 2), names=NAMES, **opts):
    from b200 import capi
    rng = np.random.default_rng(seed)
    B = len(sizes)
    surf = Surfaces(sizes, nv12, rng)
    before = surf.host()
    sc, lab, bx, ids, cnt = entries(rng, sizes, k, nc, with_ids)
    ann = capi.Annotator(nc, names=names[:nc], privacy=privacy, **opts)
    spec = an.Annotator(nc, names=names[:nc], privacy=privacy, **opts)
    dev = lambda x: None if x is None else torch.from_numpy(x).cuda()  # noqa: E731
    zo, occ, geo, totals, streams = None, None, None, None, list(range(B))
    if zones:
        streams = [int(s) for s in rng.permutation(B + 3)[:B]]
        zo = capi.Zones(B + 3, num_classes=nc)
        geo = {}
        for b, s in enumerate(streams):
            h, w = sizes[b]
            lines, polys = zs.layout(seed * 131 + s, size=(h, w), **(zones if isinstance(zones, dict) else {}))
            zo.set(s, lines, polys)
            geo[s] = zs.geometry(lines, polys)
        for _ in range(3):
            tr_ids = torch.arange(1, k + 1, dtype=torch.int32).repeat(B, 1).cuda()
            jit = torch.from_numpy(rng.uniform(-40, 40, (B, k, 4)).astype(np.float32)).cuda()
            out = zo.update(tr_ids, dev(lab), dev(bx) + jit, dev(np.full(B, k, np.int32)), streams)
        occ = out[1]
        totals = {s: zo.export(s)["line_counts"].sum(axis=1) for s in streams}
    ann.annotate(surf.frames, dev(sc), dev(lab), dev(bx), ids=dev(ids), counts=dev(cnt), streams=streams, zones=zo, occupancy=occ,
                 score_threshold=threshold, colorspace=cs if nv12 else None)
    torch.cuda.synchronize()
    got = surf.host()
    assert any(not np.array_equal(g, w_) for b in range(B) for g, w_ in zip(got[b] if nv12 else [got[b]], before[b] if nv12 else [before[b]]))
    occ = None if occ is None else occ.cpu().numpy()
    for b in range(B):
        kw = dict(scores=sc[b], labels=lab[b], boxes=bx[b], ids=None if ids is None else ids[b], count=cnt[b], threshold=threshold)
        if zones:
            kw.update(geometry=geo[streams[b]], line_totals=totals[streams[b]], occupancy=occ[b])
        surf.spec_draw(before, b, spec, cs, **kw)
    for b in range(B):
        for g, w_ in zip(got[b] if nv12 else [got[b]], before[b] if nv12 else [before[b]]):
            if not np.array_equal(g, w_):
                d = np.argwhere(g != w_)
                raise AssertionError("frame %d %s: %d bytes differ, first at %s: got %d want %d"
                                     % (b, sizes[b], len(d), tuple(d[0]), g[tuple(d[0])], w_[tuple(d[0])]))


def odd_sizes(rng, B, lo=8, hi=300):
    return [(int(rng.integers(lo, hi)), int(rng.integers(lo, hi))) for _ in range(B)]


@pytest.mark.parametrize("fmt", ["rgb", "bt601", "bt709", "bt601_full", "bt709_full"])
def test_against_spec(fmt):
    rng = np.random.default_rng(len(fmt))
    nv12 = fmt != "rgb"
    cs = fmt if nv12 else None
    check([(181, 243)], nv12, cs, seed=1, box_fill_alpha=77)
    check(odd_sizes(rng, 32, 8, 160), nv12, cs, seed=2, with_ids=False, privacy_block=8, zone_fill_alpha=0)
    check([(97, 131), (64, 64), (9, 8), (200, 77)], nv12, cs, seed=3, zones=True, label=an.LABEL_ID | an.LABEL_SCORE)


def test_many_frames_and_entries():
    rng = np.random.default_rng(5)
    check(odd_sizes(rng, 256, 8, 40), False, None, k=8, seed=6, text_scale=1)
    check([(120, 200), (64, 96)], True, "bt709", k=1024, seed=7, thickness=1, text_scale=1, privacy_block=2)


@pytest.mark.parametrize("opts", [dict(thickness=32, text_scale=8, privacy_block=64, box_fill_alpha=256, zone_thickness=32),
                                  dict(thickness=1, text_scale=1, privacy_block=2, label=0, zone_thickness=1, zone_fill_alpha=256)])
def test_limits(opts):
    check([(203, 151), (77, 300)], False, None, seed=8, zones=True, **opts)
    check([(203, 151)], True, "bt601", seed=9, zones=True, **opts)


def test_zones_at_their_limits():
    check([(260, 250)], True, "bt601_full", seed=10, zones=dict(lines=32, polygons=8, vertices=256), k=16)
    check([(130, 170)], False, None, seed=11, zones=dict(lines=32, polygons=32, vertices=64), k=16, zone_fill_alpha=255)


def test_privacy_edges_and_overlaps():
    from b200 import capi
    rng = np.random.default_rng(12)
    for nv12, cs in ((False, None), (True, "bt709")):
        surf = Surfaces([(45, 71)], nv12, rng)
        before = surf.host()
        boxes = np.array([[[30, 20, 71, 45], [50, 10, 80, 40], [-5, -5, 9, 9], [60, 0, 71, 3]]], np.float32)
        lab = np.array([[1, 1, 1, 0]], np.int32)
        sc = np.ones((1, 4), np.float32)
        ann = capi.Annotator(3, privacy=[1], privacy_block=16)
        ann.annotate(surf.frames, torch.from_numpy(sc).cuda(), torch.from_numpy(lab).cuda(), torch.from_numpy(boxes).cuda(), colorspace=cs)
        torch.cuda.synchronize()
        surf.spec_draw(before, 0, an.Annotator(3, privacy=[1], privacy_block=16), cs, scores=sc[0], labels=lab[0], boxes=boxes[0])
        for g, w_ in zip(surf.host()[0] if nv12 else [surf.host()[0]], before[0] if nv12 else [before[0]]):
            assert np.array_equal(g, w_)


def test_option_and_argument_validation():
    from b200 import capi
    ann = capi.Annotator(5)
    for name, v in (("thickness", 0), ("thickness", 33), ("text_scale", 9), ("box_fill_alpha", 257), ("label", 8),
                    ("zone_fill_alpha", -1), ("zone_thickness", 0), ("privacy_block", 12), ("privacy_block", 128), ("nope", 1)):
        with pytest.raises(RuntimeError):
            ann.set_option(name, v)
    with pytest.raises(RuntimeError, match="longer than 31"):
        ann.set_names(["x" * 32])
    with pytest.raises(RuntimeError, match="more than num_classes"):
        ann.set_names(["a"] * 6)
    with pytest.raises(RuntimeError, match="outside"):
        ann.set_privacy([5])
    with pytest.raises(RuntimeError):
        ann.set_palette(np.zeros((257, 3), np.uint8))
    f = torch.zeros(16, 16, 3, dtype=torch.uint8, device="cuda")
    s = torch.zeros(1, 2, device="cuda")
    with pytest.raises(RuntimeError, match="k must be"):
        ann.annotate([f], torch.zeros(1, 1025, device="cuda"), torch.zeros(1, 1025, dtype=torch.int32, device="cuda"),
                     torch.zeros(1, 1025, 4, device="cuda"))
    with pytest.raises(RuntimeError, match="sides"):
        ann.annotate([torch.zeros(4, 16, 3, dtype=torch.uint8, device="cuda")], s, s.int(), torch.zeros(1, 2, 4, device="cuda"))
    with pytest.raises(RuntimeError, match="CUDA"):
        ann.annotate([f.cpu()], s, s.int(), torch.zeros(1, 2, 4, device="cuda"))


def test_graph_replay_equals_eager():
    from b200 import capi
    rng = np.random.default_rng(13)
    B, k = 8, 64
    sizes = [(270, 480)] * B
    sc, lab, bx, _, _ = entries(rng, sizes, k, 6)
    sc = torch.from_numpy(sc).cuda()
    lab = torch.from_numpy(np.abs(lab)).cuda()
    bx = torch.from_numpy(bx).cuda()

    def make():
        tr = capi.Tracker(B)
        zo = capi.Zones(B, num_classes=6)
        for s in range(B):
            lines, polys = zs.layout(s, size=(270, 480))
            zo.set(s, lines, polys)
        return tr, zo, capi.Annotator(6, privacy=[3])

    def step(tr, zo, ann, frames, t):
        got = tr.update(sc, lab, bx + t, max_out=k)
        _, occ, _, _ = zo.update(got[0], got[2], got[3], got[5])
        ann.annotate(frames, got[1], got[2], got[3], ids=got[0], counts=got[5], zones=zo, occupancy=occ)

    base = torch.from_numpy(rng.integers(0, 256, (B, 270, 480, 3), dtype=np.uint8)).cuda()
    eager, graphed = base.clone(), base.clone()
    shift = torch.zeros(1, device="cuda")
    tr, zo, ann = make()
    for i in range(3):
        shift.fill_(float(i))
        step(tr, zo, ann, eager, shift)
    tr2, zo2, ann2 = make()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    shift.fill_(0.0)
    with torch.cuda.stream(s):
        step(tr2, zo2, ann2, graphed, shift)                    # frame 1 eagerly (warm-up), then capture frames 2 and 3
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step(tr2, zo2, ann2, graphed, shift)
    torch.cuda.current_stream().wait_stream(s)
    for i in (1, 2):
        shift.fill_(float(i))
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager, graphed)


def test_track_annotate():
    from b200 import capi
    from b200.config import CONFIGS
    from b200.synth import synth_state_dict
    from models.lwdetr import LWDETR
    cfg = CONFIGS["tiny"]
    model = LWDETR(cfg, compute_dtype=torch.float16).eval()
    model.load_state_dict(synth_state_dict(cfg, 1), strict=True)
    model.to("cuda")
    rng = np.random.default_rng(14)
    B = 4
    frames = [torch.from_numpy(rng.integers(0, 256, (360, 640, 3), dtype=np.uint8)).cuda() for _ in range(B)]
    nv = [torch.from_numpy(rng.integers(0, 256, (540, 640), dtype=np.uint8)).cuda() for _ in range(B)]

    def zones():
        z = capi.Zones(B, num_classes=cfg.num_classes)
        for s in range(B):
            z.set(s, *zs.layout(s, size=(360, 640)))
        return z

    for fr, cs in ((frames, None), (nv, "bt709")):
        plain = [f.clone() for f in fr]
        drawn = [f.clone() for f in fr]
        params = dict(track_thresh=0.05, low_thresh=0.01, new_track_thresh=0.05)
        tr_a, tr_b = capi.Tracker(B, **params), capi.Tracker(B, **params)
        za, zb = zones(), zones()
        ann = capi.Annotator(cfg.num_classes, privacy=[2], box_fill_alpha=40)
        da = model.track(plain, tr_a, colorspace=cs, zones=za)
        db = model.track(drawn, tr_b, colorspace=cs, zones=zb, annotate=ann)
        ref = [f.clone() for f in fr]
        ann.draw(ref, db, zones=zb, colorspace=cs)
        torch.cuda.synchronize()
        for x, y in zip(da, db):
            assert x.keys() == y.keys() and all(torch.equal(x[key], y[key]) for key in x)
        assert all(torch.equal(p, f) for p, f in zip(plain, fr))
        assert all(torch.equal(a, b) for a, b in zip(drawn, ref))
        assert any(not torch.equal(a, f) for a, f in zip(drawn, fr))


def test_zones_set_waits_for_an_annotate_that_reads_them():
    """Zones.set right after an annotate that reads the object, with no synchronisation and the stream still busy: the
    annotate draws the geometry and totals it was called with."""
    from b200 import capi
    rng = np.random.default_rng(15)
    h, w, k = 180, 260, 30
    surf = Surfaces([(h, w)], False, rng)
    before = surf.host()
    sc, lab, bx, ids, cnt = entries(rng, [(h, w)], k, 4)
    lab = np.abs(lab) % 4
    zo = capi.Zones(1, num_classes=4)
    old = zs.layout(16, size=(h, w), lines=6, polygons=6, vertices=24)
    zo.set(0, *old)
    jit = [torch.from_numpy(rng.uniform(-30, 30, (1, k, 4)).astype(np.float32)).cuda() for _ in range(3)]
    ids_t = torch.arange(1, k + 1, dtype=torch.int32)[None].cuda()
    for j in jit:
        _, occ, _, _ = zo.update(ids_t, torch.from_numpy(lab).cuda(), torch.from_numpy(bx).cuda() + j, torch.full((1,), k, dtype=torch.int32).cuda())
    totals = zo.export(0)["line_counts"].sum(axis=1)
    ann = capi.Annotator(4)
    torch.cuda._sleep(400_000_000)                                  # keeps the stream busy well past the set below
    ann.annotate(surf.frames, torch.from_numpy(sc).cuda(), torch.from_numpy(lab).cuda(), torch.from_numpy(bx).cuda(),
                 ids=torch.from_numpy(ids).cuda(), counts=torch.from_numpy(cnt).cuda(), zones=zo, occupancy=occ)
    zo.set(0, [(1, 1, 5, 5)], [[(0, 0), (3, 0), (0, 3)]])          # new, shorter geometry; clears the counters
    torch.cuda.synchronize()
    surf.spec_draw(before, 0, an.Annotator(4), None, scores=sc[0], labels=lab[0], boxes=bx[0], ids=ids[0], count=cnt[0],
                   geometry=zs.geometry(*old), line_totals=totals, occupancy=occ[0].cpu().numpy())
    assert np.array_equal(surf.host()[0], before[0])
    assert zo.export(0)["line_counts"].shape[0] == 1


def test_kernel_fill_is_what_device_zones_count():
    """The draw kernel's polygon fill against the zones kernel's own inside masks, one track per pixel centre (its box's
    bottom-centre anchor there), on every pixel off the polygon's outline."""
    from b200 import capi
    h, w = 30, 34
    ys, xs = np.mgrid[0:h, 0:w]
    boxes = np.stack([xs, ys - 0.5, xs + 1, ys + 0.5], -1).reshape(1, -1, 4).astype(np.float32)
    n = h * w
    for seed in range(3):
        poly = zs.star(17, 15, 14, 5, 5 + seed, phase=0.3 * seed) if seed < 2 else np.random.default_rng(seed).uniform(-4, 38, (11, 2))
        zo = capi.Zones(1, num_classes=1, capacity=n)
        zo.set(0, (), [poly])
        inside, _, _, _ = zo.update(torch.arange(1, n + 1, dtype=torch.int32)[None].cuda(), torch.zeros(1, n, dtype=torch.int32).cuda(),
                                    torch.from_numpy(boxes).cuda(), torch.full((1,), n, dtype=torch.int32).cuda(), max_events=0)
        counted = (inside.cpu().numpy()[0] & 1).astype(bool).reshape(h, w)
        frame = torch.zeros(h, w, 3, dtype=torch.uint8, device="cuda")
        ann = capi.Annotator(1, palette=[(255, 0, 0)], zone_fill_alpha=256, zone_thickness=1, label=0)
        one = torch.zeros(1, 1, device="cuda")
        ann.annotate([frame], one, one.int(), torch.zeros(1, 1, 4, device="cuda"), zones=zo)
        drawn = frame.cpu().numpy()[..., 0] == 255
        spec = an.Annotator(1, zone_fill_alpha=256, zone_thickness=1, label=0)
        edges = np.zeros((h, w), bool)
        for q in spec.primitives(h, w, scores=np.zeros(0, np.float32), labels=np.zeros(0, np.int32), boxes=np.zeros((0, 4), np.float32),
                                 geometry=zs.geometry((), [poly]), line_totals=[]):
            if q["kind"] == "seg":
                edges |= spec.coverage(q, h, w)
        assert counted[~edges].any() and (~counted[~edges]).any()
        assert np.array_equal(drawn[~edges], counted[~edges])
