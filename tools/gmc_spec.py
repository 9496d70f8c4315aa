"""Camera-motion estimation (lwdetr_gmc_estimate in include/lwdetr_b200.h), restated in numpy for the tests: the grey,
downscale and pyramid rule and the corner rule bit for bit, the hypothesis hash, RANSAC and the least-squares refit given
point pairs.  The Lucas-Kanade step is OpenCV's; the tests compare the kernel with cv2.calcOpticalFlowPyrLK directly.

botsort_gmc() is BoT-SORT's sparseOptFlow method written with cv2 (the reference the estimator is measured against);
textured_frame() and warp_frame() make seeded test frames whose motion is known.
"""
import numpy as np

PARAMS = dict(downscale=2, max_points=1024, quality=0.01, levels=3, window=21, iterations=30, eps=0.01, min_eig=1e-4,
              ransac_thresh=3.0, hypotheses=1024, min_inliers=10, max_height=2160, max_width=3840)
REFITS = 3
OK, FIRST_FRAME, SIZE_CHANGED, FEW_POINTS, FEW_INLIERS = 0, 1, 2, 3, 4


def params(**kw):
    bad = set(kw) - set(PARAMS)
    if bad:
        raise TypeError("unknown estimator parameters: %s" % ", ".join(sorted(bad)))
    p = dict(PARAMS)
    p.update(kw)
    for k in ("quality", "eps", "min_eig", "ransac_thresh"):
        p[k] = np.float32(p[k])
    return p


# ---------------------------------------------------------------------------------------------- grey, level 0, pyramid
def grey_rgb(rgb):
    """cv2.COLOR_RGB2GRAY of uint8 [h, w, 3]: (9798 R + 19235 G + 3735 B + 16384) >> 15."""
    c = rgb.astype(np.int32)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + 16384) >> 15).astype(np.uint8)


def level0(grey, d):
    """Box average of d x d blocks, (S + d*d // 2) // (d*d), over (h // d, w // d)."""
    h, w = grey.shape[0] // d, grey.shape[1] // d
    s = grey[:h * d, :w * d].astype(np.int32).reshape(h, d, w, d).sum(axis=(1, 3))
    return ((s + d * d // 2) // (d * d)).astype(np.uint8)


def pyr_down(img):
    """cv2.pyrDown: 5-tap [1 4 6 4 1] both ways, BORDER_REFLECT_101, (sum + 128) >> 8, size ((w + 1) // 2, (h + 1) // 2)."""
    h, w = img.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    k = np.array([1, 4, 6, 4, 1], np.int32)
    p = np.pad(img.astype(np.int32), 2, mode="reflect")
    rows = sum(k[j] * p[:, j:j + 2 * ow:2] for j in range(5))
    out = sum(k[r] * rows[r:r + 2 * oh:2, :] for r in range(5))
    return ((out + 128) >> 8).astype(np.uint8)


def geometry(h, w, p):
    """(level sizes [(h_l, w_l)], levels used, cell side, cells across, cells down) of an h x w frame."""
    d = p["downscale"]
    sizes = [(h // d, w // d)]
    for _ in range(5):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    nlev = 0
    while nlev < p["levels"] and sizes[nlev + 1][0] > p["window"] and sizes[nlev + 1][1] > p["window"]:
        nlev += 1
    h0, w0 = sizes[0]
    c = max(1, int(np.sqrt(float(h0 * w0) / p["max_points"])))
    while -(-w0 // c) * -(-h0 // c) > p["max_points"]:
        c += 1
    return sizes, nlev, c, -(-w0 // c), -(-h0 // c)


def pyramid(grey, p):
    """Levels 0..levels used of a grey frame."""
    _, nlev, _, _, _ = geometry(grey.shape[0], grey.shape[1], p)
    lv = [level0(grey, p["downscale"])]
    for _ in range(nlev):
        lv.append(pyr_down(lv[-1]))
    return lv


# ---------------------------------------------------------------------------------------------- corners
def response(img):
    """Shi-Tomasi response of every pixel: Sobel 3x3 (BORDER_REFLECT_101), products summed over 3x3 (BORDER_REFLECT_101),
    R = (Sxx + Syy) - sqrt((Sxx - Syy)^2 + 4 Sxy^2) in float64 from exact integers."""
    p = np.pad(img.astype(np.int64), 1, mode="reflect")
    dx = (p[:-2, 2:] - p[:-2, :-2]) + 2 * (p[1:-1, 2:] - p[1:-1, :-2]) + (p[2:, 2:] - p[2:, :-2])
    dy = (p[2:, :-2] - p[:-2, :-2]) + 2 * (p[2:, 1:-1] - p[:-2, 1:-1]) + (p[2:, 2:] - p[:-2, 2:])

    def box(a):
        q = np.pad(a, 1, mode="reflect")
        return sum(q[r:r + a.shape[0], c:c + a.shape[1]] for r in range(3) for c in range(3))
    sxx, sxy, syy = box(dx * dx), box(dx * dy), box(dy * dy)
    disc = (sxx - syy) ** 2 + 4 * sxy * sxy
    return (sxx + syy).astype(np.float64) - np.sqrt(disc.astype(np.float64))


def corners(img, p):
    """The corner rule on level 0: the best pixel of each c x c cell (row-major cells; lowest pixel index on ties), kept when
    R > 0 and R >= quality * max R.  Returns float32 [n, 2] (x, y) in cell order."""
    h, w = img.shape
    _, _, c, ncx, ncy = geometry(h * p["downscale"], w * p["downscale"], p)
    R = response(img)
    full = np.full((ncy * c, ncx * c), -np.inf)
    full[:h, :w] = R
    cells = full.reshape(ncy, c, ncx, c).transpose(0, 2, 1, 3).reshape(ncy, ncx, c * c)
    arg = cells.argmax(-1)
    best = np.take_along_axis(cells, arg[..., None], -1)[..., 0]
    ys = np.arange(ncy)[:, None] * c + arg // c
    xs = np.arange(ncx)[None, :] * c + arg % c
    thr = np.float64(np.float32(p["quality"])) * R.max()
    keep = (best > 0) & (best >= thr)
    return np.stack([xs[keep], ys[keep]], 1).astype(np.float32)


# ---------------------------------------------------------------------------------------------- robust fit
def _mix(x):
    x = np.asarray(x, np.uint64) & 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def hyp_hash(k):
    """H(k) = mix(k * 0x9e3779b9 + 0x7f4a7c15), uint32 arithmetic."""
    return _mix((np.asarray(k, np.uint64) * 0x9E3779B9 + 0x7F4A7C15) & 0xFFFFFFFF)


def hypothesis_pairs(H, n):
    """(i, j) of hypotheses 0..H-1 over n pairs: i = H(2h) mod n, j = H(2h + 1) mod (n - 1), plus 1 when >= i."""
    h = np.arange(H, dtype=np.uint64)
    i = (hyp_hash(2 * h) % np.uint64(n)).astype(np.int64)
    j = (hyp_hash(2 * h + 1) % np.uint64(n - 1)).astype(np.int64)
    return i, j + (j >= i)


def err2(m, P, Q):
    """Squared transfer error of pairs (P -> Q) under similarities m [..., 4], each operation rounded on its own."""
    a, b, tx, ty = (m[..., k:k + 1] for k in range(4))
    ex = ((a * P[:, 0] - b * P[:, 1]) + tx) - Q[:, 0]
    ey = ((b * P[:, 0] + a * P[:, 1]) + ty) - Q[:, 1]
    return ex * ex + ey * ey


def minimal(P, Q, i, j):
    """Similarity of the two pairs (i, j) (arrays); rows with n2 not > 0 are NaN."""
    dpx, dpy = P[j, 0] - P[i, 0], P[j, 1] - P[i, 1]
    dqx, dqy = Q[j, 0] - Q[i, 0], Q[j, 1] - Q[i, 1]
    n2 = dpx * dpx + dpy * dpy
    with np.errstate(invalid="ignore", divide="ignore"):
        a = (dqx * dpx + dqy * dpy) / n2
        b = (dqy * dpx - dqx * dpy) / n2
    tx = Q[i, 0] - (a * P[i, 0] - b * P[i, 1])
    ty = Q[i, 1] - (b * P[i, 0] + a * P[i, 1])
    m = np.stack([a, b, tx, ty], -1)
    m[~(n2 > 0)] = np.nan
    return m


def refit(P, Q, mask):
    """Least-squares similarity of the pairs under mask (centred sums), or None when degenerate."""
    if mask.sum() < 2:
        return None
    p, q = P[mask], Q[mask]
    mp, mq = p.mean(0), q.mean(0)
    pc, qc = p - mp, q - mq
    s = (pc * pc).sum()
    if not s > 0:
        return None
    a = (pc[:, 0] * qc[:, 0] + pc[:, 1] * qc[:, 1]).sum() / s
    b = (pc[:, 0] * qc[:, 1] - pc[:, 1] * qc[:, 0]).sum() / s
    return np.array([a, b, mq[0] - (a * mp[0] - b * mp[1]), mq[1] - (b * mp[0] + a * mp[1])])


def fit(P, Q, p):
    """The robust fit of float64 pairs P -> Q [n, 2] in frame pixels: (motion [4], status, inliers, best hypothesis)."""
    ident = np.array([1.0, 0.0, 0.0, 0.0])
    n = len(P)
    if n < p["min_inliers"]:
        return ident, FEW_POINTS, 0, -1
    thr = np.float64(p["ransac_thresh"]) * np.float64(p["downscale"])
    thr2 = thr * thr
    i, j = hypothesis_pairs(p["hypotheses"], n)
    m = minimal(P, Q, i, j)
    with np.errstate(invalid="ignore"):
        counts = (err2(m, P, Q) <= thr2).sum(1)
    counts[np.isnan(m[:, 0])] = -1
    best = int(np.argmax(counts))
    if counts[best] < p["min_inliers"]:
        return ident, FEW_INLIERS, 0, best
    model = m[best]
    for _ in range(REFITS):
        new = refit(P, Q, err2(model[None], P, Q)[0] <= thr2)
        if new is None:
            break
        model = new
    ninl = int((err2(model[None], P, Q)[0] <= thr2).sum())
    if ninl < p["min_inliers"]:
        return ident, FEW_INLIERS, ninl, best
    return model, OK, ninl, best


def to_frame(pts, d):
    """Level-0 pixel coordinates -> frame pixels: d * (x + 0.5) - 0.5."""
    return np.float64(d) * (np.asarray(pts, np.float64) + 0.5) - 0.5


# ---------------------------------------------------------------------------------------------- similarities
def matrix(m):
    """2 x 3 affine matrix of (a, b, tx, ty)."""
    a, b, tx, ty = m
    return np.array([[a, -b, tx], [b, a, ty]], np.float64)


def from_matrix(M):
    return np.array([M[0, 0], M[1, 0], M[0, 2], M[1, 2]], np.float64)


def similarity(angle_deg, scale, tx, ty, centre=(0.0, 0.0)):
    """(a, b, tx, ty) rotating by angle_deg and scaling about centre, then translating by (tx, ty)."""
    t = np.deg2rad(angle_deg)
    a, b = scale * np.cos(t), scale * np.sin(t)
    cx, cy = centre
    return np.array([a, b, cx - (a * cx - b * cy) + tx, cy - (b * cx + a * cy) + ty])


def corner_error(m, truth, h, w):
    """Largest distance between the images of the frame's four corners under m and under truth, in pixels."""
    c = np.array([[0, 0], [w - 1, 0], [0, h - 1], [w - 1, h - 1]], np.float64)
    ca = np.c_[c, np.ones(4)] @ matrix(m).T
    cb = np.c_[c, np.ones(4)] @ matrix(truth).T
    return float(np.sqrt(((ca - cb) ** 2).sum(1)).max())


# ---------------------------------------------------------------------------------------------- test frames
def textured_frame(seed, h, w, margin=0):
    """Seeded RGB uint8 [h + 2 margin, w + 2 margin, 3]: blobs, edges and fine noise at several scales, so corners and flow
    exist everywhere."""
    import cv2
    rng = np.random.default_rng(seed)
    H, W = h + 2 * margin, w + 2 * margin
    img = np.zeros((H, W, 3), np.float32)
    for cell in (96, 24, 6):
        g = rng.uniform(0, 255, (H // cell + 2, W // cell + 2, 3)).astype(np.float32)
        img += cv2.resize(g, (W + 2 * cell, H + 2 * cell), interpolation=cv2.INTER_CUBIC)[cell:cell + H, cell:cell + W] / 3
    for _ in range(max(8, H * W // 20000)):
        x, y = int(rng.integers(0, W)), int(rng.integers(0, H))
        r = int(rng.integers(3, 40))
        col = tuple(float(v) for v in rng.uniform(0, 255, 3))
        if rng.random() < 0.5:
            cv2.circle(img, (x, y), r, col, -1)
        else:
            cv2.rectangle(img, (x, y), (x + r, y + int(rng.integers(3, 40))), col, -1)
    return np.clip(img, 0, 255).astype(np.uint8)


def warp_frame(img, m, h, w):
    """The h x w view of img under the similarity m (frame pixels, cv2.warpAffine, bilinear, reflected border)."""
    import cv2
    return cv2.warpAffine(img, matrix(m), (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)


def moving_pair(seed, h, w, m, outlier_area=0.2):
    """(prev, cur, truth): a textured frame and its view under the similarity m, with a block of outlier_area of the frame
    pasted at a different, independent offset in both (an object moving on its own)."""
    rng = np.random.default_rng(seed + 7)
    base = textured_frame(seed, h, w)
    prev = base.copy()
    cur = warp_frame(base, m, h, w)
    if outlier_area > 0:
        bh, bw = int(h * np.sqrt(outlier_area)), int(w * np.sqrt(outlier_area))
        obj = textured_frame(seed + 1000, bh + 80, bw + 80)
        y0, x0 = int(rng.integers(0, h - bh)), int(rng.integers(0, w - bw))
        dy, dx = int(rng.integers(-30, 31)), int(rng.integers(-30, 31))
        prev[y0:y0 + bh, x0:x0 + bw] = obj[40:40 + bh, 40:40 + bw]
        y1, x1 = min(max(y0 + dy, 0), h - bh), min(max(x0 + dx, 0), w - bw)
        cur[y1:y1 + bh, x1:x1 + bw] = obj[40 + 7:40 + 7 + bh, 40 - 5:40 - 5 + bw]
    return prev, cur, m


def rgb_to_nv12(rgb):
    """Luma / chroma planes of an RGB frame (BT.601 limited range, cv2), for NV12 tests: (luma [h, w], chroma [h/2, w])."""
    import cv2
    h, w = rgb.shape[:2]
    i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
    y = i420[:h]
    u = i420[h:h + h // 4].reshape(h // 2, w // 2)
    v = i420[h + h // 4:].reshape(h // 2, w // 2)
    return y.copy(), np.stack([u, v], -1).reshape(h // 2, w).copy()


# ---------------------------------------------------------------------------------------------- BoT-SORT's method
def botsort_gmc(prev, cur, downscale=2):
    """BoT-SORT's GMC sparseOptFlow for one pair of RGB frames: grey, cv2.resize by downscale, goodFeaturesToTrack
    (1000 corners, quality 0.01, minDistance 1, blockSize 3) on the previous frame, calcOpticalFlowPyrLK with its defaults,
    estimateAffinePartial2D(RANSAC), translation times downscale.  Returns (a, b, tx, ty) or the identity."""
    import cv2

    def prep(f):
        g = cv2.cvtColor(f, cv2.COLOR_RGB2GRAY) if f.ndim == 3 else f
        h, w = g.shape
        return cv2.resize(g, (w // downscale, h // downscale)) if downscale > 1 else g
    a, b = prep(prev), prep(cur)
    kp = cv2.goodFeaturesToTrack(a, mask=None, maxCorners=1000, qualityLevel=0.01, minDistance=1, blockSize=3,
                                 useHarrisDetector=False, k=0.04)
    ident = np.array([1.0, 0.0, 0.0, 0.0])
    if kp is None:
        return ident
    nxt, st, _ = cv2.calcOpticalFlowPyrLK(a, b, kp, None)
    ok = st.reshape(-1) == 1
    if ok.sum() <= 4:
        return ident
    M, _ = cv2.estimateAffinePartial2D(kp[ok], nxt[ok], method=cv2.RANSAC)
    if M is None:
        return ident
    M = M.copy()
    M[0, 2] *= downscale
    M[1, 2] *= downscale
    return from_matrix(M)
