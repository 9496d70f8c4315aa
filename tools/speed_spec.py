"""Ground-plane position, velocity and speed per camera stream (lwdetr_speed_* in include/lwdetr_b200.h), restated in numpy
for the tests: supervision's speed estimation after the tracker, on the tracker's own outputs (ids, xyxy boxes in frame
pixels, counts), with a per-stream homography from frame pixels to the ground.

Everything is float64 with each operation rounded on its own (numpy does not fuse), in the order the header fixes.
Elementwise numpy arithmetic rounds each operation exactly as the kernel's __dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn
do, and the sums run left to right (np.cumsum accumulates in order), so the two agree bit for bit.

Also here: a synthetic road scene seen by a pinhole camera, with the true ground velocity of every object.
"""
import numpy as np

MAX_CAPACITY, MAX_WINDOW, MAX_OUT = 4096, 64, 1024
BOTTOM_CENTER = 7
DEFAULTS = dict(capacity=1024, window=30, min_samples=15, forget_after=30, anchor=BOTTOM_CENTER, frame_rate=30.0)


def params(**kw):
    """The parameters with lwdetr_speed_create's defaults, validated as it does."""
    bad = set(kw) - set(DEFAULTS)
    if bad:
        raise TypeError("unknown speed parameters: %s" % ", ".join(sorted(bad)))
    p = dict(DEFAULTS)
    p.update(kw)
    if not 1 <= p["capacity"] <= MAX_CAPACITY or not 2 <= p["window"] <= MAX_WINDOW or not 2 <= p["min_samples"] <= p["window"] \
            or p["forget_after"] < 0 or not 0 <= p["anchor"] < 9 or not (np.isfinite(p["frame_rate"]) and p["frame_rate"] > 0):
        raise ValueError("speed parameters out of range: %s" % p)
    return p


def anchors(boxes, which):
    """Anchor `which` (0..8) of fp32 xyxy boxes [n, 4], widened to float64: (x, y) arrays (the zones' rule)."""
    b = np.asarray(boxes, np.float32).astype(np.float64).reshape(-1, 4)
    row, col = divmod(which, 3)
    x = (b[:, 0], (b[:, 0] + b[:, 2]) * 0.5, b[:, 2])[col]
    y = (b[:, 1], (b[:, 1] + b[:, 3]) * 0.5, b[:, 3])[row]
    return x, y


def check_homography(H):
    """lwdetr_speed_set's checks: H float64 [3, 3], finite, determinant (in the header's order) neither 0 nor non-finite."""
    h = np.asarray(H, np.float64)
    if h.shape != (3, 3) or not np.isfinite(h).all():
        raise ValueError("the homography must be a finite [3, 3] array")
    f = [float(v) for v in h.reshape(-1)]
    det = f[0] * (f[4] * f[8] - f[5] * f[7]) - f[1] * (f[3] * f[8] - f[5] * f[6]) + f[2] * (f[3] * f[7] - f[4] * f[6])
    if det == 0.0 or not np.isfinite(det):
        raise ValueError("the homography is singular")
    return h.copy()


def project(H, x, y):
    """(x, y) pixels -> (X, Y, valid): w = (h6 x + h7 y) + h8, X = ((h0 x + h1 y) + h2) / w, Y likewise; valid iff w > 0 and
    X, Y finite."""
    h = np.asarray(H, np.float64).reshape(-1)
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        w = (h[6] * x + h[7] * y) + h[8]
        X = ((h[0] * x + h[1] * y) + h[2]) / w
        Y = ((h[3] * x + h[4] * y) + h[5]) / w
    return X, Y, (w > 0) & np.isfinite(X) & np.isfinite(Y)


def fit(samples, H, min_samples):
    """The contract's least-squares fit over a ring's samples [n, 3] (t, x, y), oldest first: (n valid, vX, vY, speed), the
    last three NaN without an estimate."""
    s = np.asarray(samples, np.float64).reshape(-1, 3)
    X, Y, ok = project(H, s[:, 1], s[:, 2])
    t, X, Y = s[ok, 0], X[ok], Y[ok]
    n = len(t)
    if n == 0:
        return 0, np.nan, np.nan, np.nan
    tau = t - t[-1]
    mt, mx, my = np.cumsum(tau)[-1] / n, np.cumsum(X)[-1] / n, np.cumsum(Y)[-1] / n
    d = tau - mt
    stt, stx, sty = np.cumsum(d * d)[-1], np.cumsum(d * (X - mx))[-1], np.cumsum(d * (Y - my))[-1]
    if n < min_samples or not stt > 0:
        return n, np.nan, np.nan, np.nan
    vx, vy = stx / stt, sty / stt
    return n, vx, vy, np.sqrt(vx * vx + vy * vy)


class Stream:
    """One stream's homography, clock, records (one ring per track id) and counters."""

    def __init__(self, p):
        self.p = p
        self.H = np.eye(3)
        self.reset()

    def reset(self):
        """Frame back to 1, no records, counters zero, last_t -inf; H kept."""
        self.frame, self.overflow, self.clock_errors, self.last_t = 1, 0, 0, -np.inf
        self.records = {}

    def set(self, H):
        """A new homography; the history is kept."""
        self.H = check_homography(H)

    def update(self, ids, boxes, count, t=None, max_out=None):
        """One frame: the tracker's ids int32 [max_out], boxes fp32 [max_out, 4] and count; t the frame's timestamp (None:
        frame / frame_rate) -> (kin fp32 [max_out, 5] = (X, Y, vX, vY, speed), samples int32 [max_out])."""
        p, frame = self.p, self.frame
        ids = np.asarray(ids, np.int32)
        boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
        max_out = len(ids) if max_out is None else max_out
        t = np.float64(frame) / np.float64(p["frame_rate"]) if t is None else np.float64(t)
        clock_ok = bool(np.isfinite(t) and t > self.last_t)
        if clock_ok:
            self.last_t = t
        else:
            self.clock_errors += 1
        present, seen = [], set()
        for j in range(max(0, min(int(count), max_out))):
            i = int(ids[j])
            if i <= 0 or not np.isfinite(boxes[j]).all() or i in seen:
                continue
            seen.add(i)
            present.append(j)
        kin = np.full((max_out, 5), np.nan, np.float32)
        samples = np.zeros(max_out, np.int32)
        ax, ay = anchors(boxes[present], p["anchor"])
        X, Y, ok = project(self.H, ax, ay)
        free = p["capacity"] - len(self.records)
        for q, j in enumerate(present):
            if ok[q]:
                kin[j, 0], kin[j, 1] = X[q], Y[q]
            tid = int(ids[j])
            rec = self.records.get(tid)
            if rec is None:
                if free == 0:
                    self.overflow += 1
                    continue
                free -= 1
                rec = self.records[tid] = dict(ring=[], last_seen=frame)
            if clock_ok:
                rec["ring"].append((t, ax[q], ay[q]))
                del rec["ring"][:-p["window"]]
            rec["last_seen"] = frame
            n, vx, vy, sp = fit(rec["ring"], self.H, p["min_samples"])
            kin[j, 2:] = vx, vy, sp
            samples[j] = n
        for tid in sorted(self.records):
            if frame - self.records[tid]["last_seen"] > p["forget_after"]:
                del self.records[tid]
        self.frame += 1
        return kin, samples

    def export(self):
        """lwdetr_speed_export's result as SpeedEstimator.export gives it, the records in ascending id."""
        ids = sorted(self.records)
        return dict(frame=self.frame, records=len(ids), overflow=self.overflow, clock_errors=self.clock_errors,
                    last_t=float(self.last_t), homography=self.H.copy(), ids=np.array(ids, np.int32),
                    last_seen=np.array([self.records[i]["last_seen"] for i in ids], np.int32),
                    samples=[np.array(self.records[i]["ring"], np.float64).reshape(-1, 3) for i in ids])


def endpoint_speed(samples, H, fps):
    """supervision's speed-estimation example on one track's samples [n, 3] (t, x, y), oldest first: the distance between
    the first and the last ground y over len / fps seconds."""
    s = np.asarray(samples, np.float64).reshape(-1, 3)
    _, Y, _ = project(H, s[:, 1], s[:, 2])
    return abs(Y[0] - Y[-1]) / (len(s) / fps)


# ---------------------------------------------------------------------------------------------- synthetic scenes
def camera(f=1500.0, height=10.0, pitch_deg=25.0, size=(1080, 1920)):
    """A pinhole camera `height` metres above a flat road, looking along +Y and pitched down by pitch_deg: dict with P, the
    3x4 world (X, Y, Z metres, Z up) -> pixel projection, and H, the float64 homography from frame pixels to the ground
    (X, Y), scaled so that |H[2, 2]| = 1 with w > 0 on the ground in front of the camera (w is 1 / depth there before the
    scaling)."""
    th = np.deg2rad(pitch_deg)
    K = np.array([[f, 0, size[1] / 2], [0, f, size[0] / 2], [0, 0, 1]])
    R = np.array([[1.0, 0.0, 0.0], [0.0, -np.sin(th), -np.cos(th)], [0.0, np.cos(th), -np.sin(th)]])   # rows: image x, y, depth
    C = np.array([0.0, 0.0, height])
    P = K @ np.hstack([R, (-R @ C)[:, None]])
    G = P[:, [0, 1, 3]]                              # the ground plane Z = 0 -> pixels
    H = np.linalg.inv(G)
    return dict(P=P, H=H / abs(H[2, 2]), size=size)


def to_pixels(P, pts):
    """World points [..., 3] -> pixels [..., 2] (float64)."""
    pts = np.asarray(pts, np.float64)
    h = pts @ P[:, :3].T + P[:, 3]
    return h[..., :2] / h[..., 2:]


def road_scene(seed, objects=200, frames=36, sigma=0.0, fps=30.0, speeds=(3.0, 35.0), cam=None, integer=False):
    """Objects moving on the ground at constant velocities of speeds[0]..speeds[1] m/s with random headings, seen by
    `cam` (default camera()) at fps.  Each box is (foot_x - w/2, top, foot_x + w/2, foot_y): the foot point is the object's
    ground point projected, the top its point 1.6 m up, w 0.4 of the height; each edge gets N(0, sigma) px of noise,
    then the box is rounded to fp32 (the only error without noise).  Every object's foot point stays inside the frame.
    Returns (boxes fp32 [frames, objects, 4], velocity float64 [objects, 2] in m/s, cam)."""
    cam = camera() if cam is None else cam
    rng = np.random.default_rng(seed)
    Hh, Ww = cam["size"]
    t = np.arange(frames) / fps
    vel, feet, tops = [], [], []
    while len(vel) < objects:
        sp, hd = rng.uniform(*speeds), rng.uniform(0, 2 * np.pi)
        v = sp * np.array([np.cos(hd), np.sin(hd)])
        mid = np.array([rng.uniform(-12, 12), rng.uniform(20, 60)])
        g = mid + (t - t[-1] / 2)[:, None] * v
        ground = np.concatenate([g, np.zeros((frames, 1))], 1)
        foot = to_pixels(cam["P"], ground)
        if not ((foot[:, 0] > 5) & (foot[:, 0] < Ww - 5) & (foot[:, 1] > 5) & (foot[:, 1] < Hh - 5)).all():
            continue
        vel.append(v)
        feet.append(foot)
        tops.append(to_pixels(cam["P"], ground + np.array([0.0, 0.0, 1.6])))
    feet, tops = np.stack(feet, 1), np.stack(tops, 1)      # [frames, objects, 2]
    h = feet[..., 1] - tops[..., 1]
    w = 0.4 * h
    boxes = np.stack([feet[..., 0] - w / 2, tops[..., 1], feet[..., 0] + w / 2, feet[..., 1]], -1)
    if sigma > 0:
        boxes = boxes + rng.normal(0, sigma, boxes.shape)
    return boxes.astype(np.float32), np.array(vel), cam


def estimate_scene(boxes, H, timestamps=None, **kw):
    """Runs one spec stream over a road_scene's boxes (ids 1..objects, every object present every frame): the last frame's
    kin [objects, 5] and samples, and the stream."""
    frames, n, _ = boxes.shape
    s = Stream(params(**kw))
    s.set(H)
    ids = np.arange(1, n + 1, dtype=np.int32)
    for f in range(frames):
        kin, samples = s.update(ids, boxes[f], n, None if timestamps is None else timestamps[f])
    return kin, samples, s
