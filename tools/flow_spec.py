"""Per-object flow (lwdetr_track_flow's flow in include/lwdetr_b200.h), restated in numpy for the tests: the Median Flow
tracker's seeds, forward-backward error, NCC, selection, medians, box and status for one track, taking the Lucas-Kanade
results as input (the tests feed them from cv2.calcOpticalFlowPyrLK or from the kernel's export).

Every float64 operation is rounded on its own (numpy does not fuse), in the header's order.

sprite_scene() renders textured sprites moving and scaling over a textured background, for the accuracy tests and the
benchmark.
"""
import numpy as np

OK, FEW_POINTS, FB, SCALE, SMALL, SKIPPED, NO_PREVIOUS = range(7)
DEFAULTS = dict(grid=10, window=15, iterations=30, eps=0.01, min_eig=1e-4, ncc_window=11, min_points=8, fb_max=10.0, scale_min=0.5,
                scale_max=2.0, max_tracks=256)


def params(**kw):
    bad = set(kw) - set(DEFAULTS)
    if bad:
        raise TypeError("unknown flow parameters: %s" % ", ".join(sorted(bad)))
    p = dict(DEFAULTS)
    p.update(kw)
    for k in ("eps", "min_eig", "fb_max", "scale_min", "scale_max"):
        p[k] = np.float32(p[k])
    return p


def seeds(mean, grid, d):
    """The grid x grid seeds (level-0 float32 [grid^2, 2], q = k grid + i) of a state (cx, cy, a, h, ...)."""
    cx, cy, a, h = (np.float64(v) for v in mean[:4])
    w = a * h
    x1 = cx - w * 0.5
    y1 = cy - h * 0.5
    g = np.arange(grid, dtype=np.float64) + 0.5
    xf = x1 + (g * w) / np.float64(grid)
    yf = y1 + (g * h) / np.float64(grid)
    X, Y = np.meshgrid(xf, yf)
    d = np.float64(d)
    return np.stack([((X + 0.5) / d - 0.5).reshape(-1), ((Y + 0.5) / d - 0.5).reshape(-1)], 1).astype(np.float32)


def to_frame(pts, d):
    return np.float64(d) * (np.asarray(pts, np.float32).astype(np.float64) + 0.5) - 0.5


def _refl(p, n):
    if n == 1:
        return np.zeros_like(p)
    p = np.abs(p)
    p = p % (2 * n - 2)
    return np.where(p >= n, 2 * n - 2 - p, p)


def ncc(prev0, cur0, p, q, win):
    """NCC of the win x win patches around round(p) in prev0 and round(q) in cur0 (round half to even, reflected)."""
    H, W = prev0.shape
    hw = win // 2
    o = np.arange(-hw, hw + 1)
    a = prev0[np.ix_(_refl(int(np.rint(p[1])) + o, H), _refl(int(np.rint(p[0])) + o, W))].astype(np.int64)
    b = cur0[np.ix_(_refl(int(np.rint(q[1])) + o, H), _refl(int(np.rint(q[0])) + o, W))].astype(np.int64)
    n = win * win
    s1, s2 = int(a.sum()), int(b.sum())
    va, vb = n * int((a * a).sum()) - s1 * s1, n * int((b * b).sum()) - s2 * s2
    cv = n * int((a * b).sum()) - s1 * s2
    if va <= 0 or vb <= 0:
        return -1.0
    return np.float64(cv) / np.sqrt(np.float64(va) * np.float64(vb))


def lower_median(v):
    v = np.sort(np.asarray(v, np.float64), kind="stable")
    return v[(len(v) - 1) // 2]


def measure(mean, seed, fwd, bwd, valid, prev0, cur0, p, d):
    """One track: (status, dx, dy, s, z [4], fb [g2], ncc [g2]) from its state (cx, cy, a, h, ...), the seeds, the forward and
    backward level-0 points (float32 [g2, 2]), their validity and the two level-0 images; NaN where the header leaves it."""
    nan = np.float64(np.nan)
    P, Q, Bk = to_frame(seed, d), to_frame(fwd, d), to_frame(bwd, d)
    valid = np.asarray(valid, bool)
    g2 = len(seed)
    fb = np.full(g2, nan)
    nc = np.full(g2, nan)
    for i in np.nonzero(valid)[0]:
        e = Bk[i] - P[i]
        fb[i] = np.sqrt(e[0] * e[0] + e[1] * e[1])
        nc[i] = ncc(prev0, cur0, seed[i], fwd[i], p["ncc_window"])
    dx = dy = s = nan
    z = np.full(4, nan)
    mfb = lower_median(fb[valid]) if valid.any() else nan
    mnc = lower_median(nc[valid]) if valid.any() else nan
    sel = np.nonzero(valid & (fb <= mfb) & (nc >= mnc))[0]
    if len(sel) < p["min_points"]:
        return FEW_POINTS, dx, dy, s, z, fb, nc
    if mfb > np.float64(p["fb_max"]):
        return FB, dx, dy, s, z, fb, nc
    dx = lower_median(Q[sel, 0] - P[sel, 0])
    dy = lower_median(Q[sel, 1] - P[sel, 1])
    ratios = []
    for a in range(len(sel)):
        for b in range(a + 1, len(sel)):
            i, j = sel[a], sel[b]
            ep = P[j] - P[i]
            dp = np.sqrt(ep[0] * ep[0] + ep[1] * ep[1])
            if dp > 0:
                eq = Q[j] - Q[i]
                ratios.append(np.sqrt(eq[0] * eq[0] + eq[1] * eq[1]) / dp)
    s = lower_median(ratios) if ratios else nan
    if not (np.isfinite(s) and np.float64(p["scale_min"]) <= s <= np.float64(p["scale_max"])):
        return SCALE, dx, dy, s, z, fb, nc
    m = np.asarray(mean, np.float64)
    h = m[3] * s
    z = np.array([m[0] + dx, m[1] + dy, m[2], h])
    two = 2.0 * np.float64(d)
    if not (m[2] * h >= two and h >= two):
        return SMALL, dx, dy, s, z, fb, nc
    return OK, dx, dy, s, z, fb, nc


def box_of(z):
    """xyxy float64 of an xyah state or measurement (the tracker's box rule)."""
    cx, cy, a, h = (np.float64(v) for v in z[:4])
    w = a * h
    x1 = cx - w / 2
    y1 = cy - h / 2
    return np.array([x1, y1, x1 + w, y1 + h])


def sprite_scene(seed, frames, objects=6, size=(1080, 1920), max_step=8.0, scale=(0.97, 1.03), occluders=0, camera=None,
                 flat=0):
    """Seeded textured sprites (gmc_spec.textured_frame) on a textured background: each sprite translates by up to max_step
    px and scales by a factor in `scale` per frame on its own path.  occluders: that many flat grey bars sweeping across the
    frame in front of the sprites; flat: that many of the sprites are texture-less (one grey level).  camera: a similarity
    (a, b, tx, ty) applied to the background per frame (about the frame origin), or None.  Returns (frames uint8 [frames,
    h, w, 3], boxes float64 [frames, objects, 4] xyxy, occluded bool [frames, objects]: a sprite an occluder or a sprite drawn
    after it overlaps)."""
    import cv2
    import gmc_spec as gs
    rng = np.random.default_rng(seed)
    H, W = size
    bg = gs.textured_frame(seed, H, W, margin=64)
    tex = [gs.textured_frame(seed * 131 + 7 + k, 320, 320) for k in range(objects)]
    for k in range(flat):
        tex[k] = np.full_like(tex[k], 128)
    st = []
    for _ in range(objects):
        h = rng.uniform(0.11, 0.22) * H
        w = h * rng.uniform(0.6, 1.3)
        st.append(dict(cx=rng.uniform(w, W - w), cy=rng.uniform(h, H - h), w=w, h=h, v=rng.uniform(-max_step, max_step, 2) * 0.7,
                       sv=rng.uniform(*scale)))
    occ = [dict(x=rng.uniform(0, W), v=rng.uniform(-30, 30), w=rng.uniform(60, 160)) for _ in range(occluders)]
    cam = np.array([1.0, 0.0, 0.0, 0.0])
    out = np.zeros((frames, H, W, 3), np.uint8)
    boxes = np.zeros((frames, objects, 4))
    hidden = np.zeros((frames, objects), bool)
    for f in range(frames):
        if f > 0:
            if camera is not None:
                a, b, tx, ty = camera
                ca, cb, ctx, cty = cam
                cam = np.array([a * ca - b * cb, b * ca + a * cb, (a * ctx - b * cty) + tx, (b * ctx + a * cty) + ty])
            for o in st:
                o["v"] = np.clip(o["v"] + rng.normal(0, 0.8, 2), -max_step, max_step)
                o["cx"] += o["v"][0]
                o["cy"] += o["v"][1]
                if rng.random() < 0.1:
                    o["sv"] = rng.uniform(*scale)
                if not (0.055 * H < o["h"] * o["sv"] < 0.37 * H):
                    o["sv"] = 1.0 / o["sv"]
                o["w"] *= o["sv"]
                o["h"] *= o["sv"]
                o["cx"] = np.clip(o["cx"], o["w"] / 2 + 20, W - o["w"] / 2 - 20)
                o["cy"] = np.clip(o["cy"], o["h"] / 2 + 20, H - o["h"] / 2 - 20)
            for c in occ:
                c["x"] = (c["x"] + c["v"]) % W
        M = np.array([[cam[0], -cam[1], cam[2] - 64], [cam[1], cam[0], cam[3] - 64]])
        img = cv2.warpAffine(bg, M, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)
        for k, o in enumerate(st):
            # the sprite's texture mapped onto its box (sub-pixel placement by an affine warp)
            sx, sy = o["w"] / 320.0, o["h"] / 320.0
            x1, y1 = o["cx"] - o["w"] / 2, o["cy"] - o["h"] / 2
            A = np.array([[sx, 0, x1 - 0.5 + 0.5 * sx], [0, sy, y1 - 0.5 + 0.5 * sy]])
            spr = cv2.warpAffine(tex[k], A, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
            msk = cv2.warpAffine(np.full((320, 320), 255, np.uint8), A, (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT)
            m = msk.astype(np.float32)[..., None] / 255.0
            img = (img * (1 - m) + spr * m + 0.5).astype(np.uint8)
            boxes[f, k] = (x1, y1, x1 + o["w"], y1 + o["h"])
        for c in occ:
            a0, a1 = int(c["x"]), int(c["x"] + c["w"])
            img[:, max(a0, 0):min(a1, W)] = 90
            for k in range(objects):
                bx = boxes[f, k]
                if bx[2] > a0 and bx[0] < a1:
                    hidden[f, k] = True
        for k in range(objects):                 # a sprite drawn later covers an earlier one
            b = boxes[f, k]
            for j in range(k + 1, objects):
                c = boxes[f, j]
                if min(b[2], c[2]) > max(b[0], c[0]) and min(b[3], c[3]) > max(b[1], c[1]):
                    hidden[f, k] = True
        out[f] = img
    return out, boxes, hidden
