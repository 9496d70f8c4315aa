"""Drawing into frames (lwdetr_annotator_* / lwdetr_annotate in include/lwdetr_b200.h), restated in numpy for the tests.

A frame is drawn as the header's primitive list, in painter's order: privacy, polygon fills, polygon edges, lines, box fills,
box outlines, labels, line texts, polygon texts.  Every primitive has a colour, an alpha and a set of covered pixels; the
segment and polygon tests are float64 with each operation rounded on its own, as numpy's elementwise arithmetic does, so
the kernel (csrc/annotate.cu) and this restatement agree bit for bit.  The font is read from csrc/font5x7.cuh, where it is
defined; there is no second copy of it here.
"""
import os
import re

import numpy as np

import yuv_spec
import zone_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FONT_PATH = os.path.join(ROOT, "lw-detr_b200", "csrc", "font5x7.cuh")

LABEL_NAME, LABEL_ID, LABEL_SCORE = 1, 2, 4
DEFAULTS = dict(thickness=2, text_scale=2, box_fill_alpha=0, label=7, zone_fill_alpha=64, zone_thickness=2, privacy_block=16)
RANGES = dict(thickness=(1, 32), text_scale=(1, 8), box_fill_alpha=(0, 256), label=(0, 7), zone_fill_alpha=(0, 256),
              zone_thickness=(1, 32))
PRIVACY_BLOCKS = (2, 4, 8, 16, 32, 64)
DEFAULT_PALETTE = np.array([(230, 25, 75), (60, 180, 75), (255, 225, 25), (0, 130, 200), (245, 130, 48), (145, 30, 180),
                            (70, 240, 240), (240, 50, 230), (210, 245, 60), (250, 190, 212), (0, 128, 128), (220, 190, 255),
                            (170, 110, 40), (255, 250, 200), (128, 0, 0), (170, 255, 195)], np.uint8)
# colorspace -> (kYR, kYG, kYB, kUR, kUG, kUB, kVR, kVG, kVB): round(2^16 m), m the inverse of each yuv_spec row
RGB2YUV = {0: (16840, 33058, 6405, -9713, -19068, 28781, 28781, -24110, -4671),
           1: (11966, 40254, 4064, -6596, -22189, 28784, 28784, -26145, -2639),
           2: (19595, 38470, 7471, -11058, -21710, 32768, 32768, -27439, -5329),
           3: (13933, 46871, 4732, -7509, -25259, 32768, 32768, -29763, -3005)}
MAX_COORD = 1 << 20


def read_font(path=FONT_PATH):
    """The 5x7 font of the C header: uint8 [95, 7], bit 4 of a row the leftmost column."""
    with open(path) as f:
        src = f.read()
    body = re.search(r"kFont5x7\s*\[[^\]]*\]\s*\[[^\]]*\]\s*=\s*\{(.*?)\n\};", src, re.S).group(1)
    rows = [[int(v, 16) for v in re.findall(r"0x[0-9A-Fa-f]+", g)] for g in re.findall(r"\{([^{}]*)\}", body)]
    return np.array(rows, np.uint8)


FONT = read_font()


def options(**kw):
    """The option block with the defaults, validated as lwdetr_annotator_set_option does."""
    o = dict(DEFAULTS)
    for k, v in kw.items():
        if k not in DEFAULTS:
            raise ValueError("unknown option %s" % k)
        if k == "privacy_block" and v not in PRIVACY_BLOCKS or k != "privacy_block" and not RANGES[k][0] <= v <= RANGES[k][1]:
            raise ValueError("option %s out of range: %r" % (k, v))
        o[k] = int(v)
    return o


def rgb_to_yuv(rgb, colorspace):
    """Palette colours uint8 [..., 3] -> (Y, Cb, Cr) uint8 [..., 3] by the header's integer table."""
    k = RGB2YUV[yuv_spec.code(colorspace)]
    c = np.asarray(rgb, np.int64)
    R, G, B = c[..., 0], c[..., 1], c[..., 2]
    off = 16 if yuv_spec.COEFFS[yuv_spec.code(colorspace)][5] else 0
    Y = ((k[0] * R + k[1] * G + k[2] * B + (1 << 15)) >> 16) + off
    U = ((k[3] * R + k[4] * G + k[5] * B + (1 << 15)) >> 16) + 128
    V = ((k[6] * R + k[7] * G + k[8] * B + (1 << 15)) >> 16) + 128
    return np.clip(np.stack([Y, U, V], -1), 0, 255).astype(np.uint8)


def grey(c):
    return (9798 * int(c[0]) + 19235 * int(c[1]) + 3735 * int(c[2]) + 16384) >> 15


def text_colour(c):
    return (0, 0, 0) if grey(c) >= 128 else (255, 255, 255)


def rect(box, h, w):
    """lwdetr_crops' rectangle of an fp32 xyxy box: (x0, y0, x1, y1), or None when it is not drawn."""
    b = np.asarray(box, np.float32)
    if not np.isfinite(b).all():
        return None
    x0, y0, x1, y1 = (int(min(max(np.floor(v), 0), n)) for v, n in zip(b, (w, h, w, h)))
    return (x0, y0, x1, y1) if x1 > x0 and y1 > y0 else None


def score_text(score):
    p = int(min(max(np.floor(np.float32(score) * np.float32(100) + np.float32(0.5)), 0), 100))
    return "1.00" if p == 100 else "0.%02d" % p


def label_text(mask, name, label, id_, score):
    parts = []
    if mask & LABEL_NAME:
        parts.append(name if name else str(label))
    if mask & LABEL_ID and id_ is not None:
        parts.append("#%d" % id_)
    if mask & LABEL_SCORE:
        parts.append(score_text(score))
    return " ".join(parts)


def text_prims(text, colour, ox, oy, s, h, w):
    """Background and glyph primitives of a text at (ox, oy)."""
    box = (max(ox, 0), max(oy, 0), min(ox + 6 * s * len(text), w), min(oy + 8 * s, h))
    return [dict(kind="fill", box=box, rgb=tuple(colour), alpha=256),
            dict(kind="text", box=box, rgb=text_colour(colour), alpha=256, origin=(ox, oy), text=text)]


class Annotator:
    """The object: options, names, palette and privacy set, as the C setters leave them."""

    def __init__(self, num_classes, names=None, palette=None, privacy=(), **opts):
        if not 1 <= num_classes <= 1024:
            raise ValueError("num_classes must be in [1, 1024]")
        self.num_classes = num_classes
        self.opts = options(**opts)
        self.names = [""] * num_classes
        if names is not None:
            names = list(names)
            if len(names) > num_classes or any(len(n) > 31 for n in names):
                raise ValueError("at most num_classes names of at most 31 characters")
            self.names[:len(names)] = names
        self.palette = DEFAULT_PALETTE if palette is None else np.asarray(palette, np.uint8).reshape(-1, 3)
        if not 1 <= len(self.palette) <= 256:
            raise ValueError("a palette has 1 to 256 colours")
        self.privacy = set(int(c) for c in privacy)
        if any(not 0 <= c < num_classes for c in self.privacy):
            raise ValueError("privacy classes must be in [0, num_classes)")

    def colour(self, i):
        return tuple(int(v) for v in self.palette[int(i) % len(self.palette)])

    def primitives(self, h, w, scores, labels, boxes, ids=None, count=None, threshold=0.0, geometry=None, line_totals=None,
                   occupancy=None):
        """The frame's primitive list in painter's order.  geometry: (lines [L, 4], polygons list of [n, 2]) or None;
        line_totals: (in, out) per line; occupancy: per polygon, or None."""
        o = self.opts
        s = o["text_scale"]
        k = len(scores)
        count = k if count is None else min(int(count), k)
        priv, fills, outlines, labs = [], [], [], []
        for j in range(count):
            if not np.float32(scores[j]) >= np.float32(threshold):
                continue
            r = rect(boxes[j], h, w)
            if r is None:
                continue
            lab = int(labels[j])
            known = 0 <= lab < self.num_classes
            if known and lab in self.privacy:
                priv.append(dict(kind="priv", box=r))
                continue
            c = self.colour(ids[j] if ids is not None else lab)
            if o["box_fill_alpha"] > 0:
                fills.append(dict(kind="fill", box=r, rgb=c, alpha=o["box_fill_alpha"]))
            outlines.append(dict(kind="outline", box=r, rgb=c, alpha=256))
            if o["label"]:
                t = label_text(o["label"], self.names[lab] if known else "", lab, None if ids is None else int(ids[j]), scores[j])
                if t:
                    oy = r[1] - 8 * s if r[1] - 8 * s >= 0 else r[1]
                    labs += text_prims(t, c, r[0], oy, s, h, w)
        pf, edges, lines, texts = [], [], [], []
        if geometry is not None:
            ln, polys = geometry
            rad = o["zone_thickness"] * 0.5
            for p, poly in enumerate(polys):
                poly = np.asarray(poly, np.float64)
                c = self.colour(p)
                if o["zone_fill_alpha"] > 0:
                    pf.append(dict(kind="poly", box=(0, 0, w, h), rgb=c, alpha=o["zone_fill_alpha"], poly=poly))
                for i in range(len(poly)):
                    seg = (*poly[i], *poly[(i + 1) % len(poly)])
                    edges.append(dict(kind="seg", box=seg_box(seg, rad, h, w), rgb=c, alpha=256, seg=seg, r=rad))
            for l, seg in enumerate(ln):
                lines.append(dict(kind="seg", box=seg_box(seg, rad, h, w), rgb=self.colour(l), alpha=256, seg=tuple(seg), r=rad))
            for l, seg in enumerate(ln):
                ox = int(min(max(np.floor((seg[0] + seg[2]) * 0.5), -MAX_COORD), MAX_COORD))
                oy = int(min(max(np.floor((seg[1] + seg[3]) * 0.5), -MAX_COORD), MAX_COORD))
                texts += text_prims("in %d out %d" % tuple(line_totals[l]), self.colour(l), ox, oy, s, h, w)
            if occupancy is not None:
                for p, poly in enumerate(polys):
                    ox, oy = (int(min(max(np.floor(v), -MAX_COORD), MAX_COORD)) for v in poly[0])
                    texts += text_prims(str(int(occupancy[p])), self.colour(p), ox, oy, s, h, w)
        return priv + pf + edges + lines + fills + outlines + labs + texts

    def coverage(self, p, h, w):
        """bool [h, w]: the pixels primitive p covers."""
        x0, y0, x1, y1 = p["box"]
        m = np.zeros((h, w), bool)
        if x1 <= x0 or y1 <= y0:
            return m
        ys, xs = np.mgrid[y0:y1, x0:x1]
        kind = p["kind"]
        if kind in ("priv", "fill"):
            c = np.ones(ys.shape, bool)
        elif kind == "outline":
            t = self.opts["thickness"]
            c = (xs < x0 + t) | (xs >= x1 - t) | (ys < y0 + t) | (ys >= y1 - t)
        elif kind == "seg":
            c = segment_covers(xs, ys, p["seg"], p["r"])
        elif kind == "poly":
            c = zone_spec.inside_polygon(xs.ravel() + 0.5, ys.ravel() + 0.5, p["poly"]).reshape(xs.shape)
        else:
            c = text_covers(xs, ys, p["origin"], p["text"], self.opts["text_scale"])
        m[y0:y1, x0:x1] = c
        return m

    def draw_rgb(self, img, **entries):
        """img uint8 [h, w, 3] drawn in place (a copy is the caller's choice); entries as primitives() takes them."""
        h, w = img.shape[:2]
        prims = self.primitives(h, w, **entries)
        priv = [p for p in prims if p["kind"] == "priv"]
        if priv:
            cov = np.zeros((h, w), bool)
            for p in priv:
                cov |= self.coverage(p, h, w)
            for c in range(3):
                img[..., c] = pixelate(img[..., c], cov, self.opts["privacy_block"])
        for p in prims:
            if p["kind"] == "priv":
                continue
            cov = self.coverage(p, h, w)
            a = p["alpha"]
            for c in range(3):
                ch = img[..., c]
                ch[cov] = blend(ch[cov], p["rgb"][c], a)
        return img

    def draw_nv12(self, luma, chroma, colorspace, **entries):
        """luma uint8 [h, w], chroma [ceil(h/2), 2 ceil(w/2)] drawn in place."""
        h, w = luma.shape
        ch, cw = (h + 1) // 2, (w + 1) // 2
        U, V = chroma[:, 0::2], chroma[:, 1::2]
        prims = self.primitives(h, w, **entries)
        priv = [p for p in prims if p["kind"] == "priv"]
        if priv:
            cov = np.zeros((h, w), bool)
            for p in priv:
                cov |= self.coverage(p, h, w)
            luma[...] = pixelate(luma, cov, self.opts["privacy_block"])
            ccov = cov[0::2, 0::2]
            U[...] = pixelate(U, ccov, self.opts["privacy_block"] // 2)
            V[...] = pixelate(V, ccov, self.opts["privacy_block"] // 2)
        for p in prims:
            if p["kind"] == "priv":
                continue
            cov = self.coverage(p, h, w)
            if not cov.any():
                continue
            yuv = rgb_to_yuv(np.array(p["rgb"], np.uint8), colorspace)
            a = p["alpha"]
            luma[cov] = blend(luma[cov], yuv[0], a)
            padded = np.zeros((2 * ch, 2 * cw), np.int64)
            padded[:h, :w] = cov
            n = padded.reshape(ch, 2, cw, 2).sum(axis=(1, 3))
            sel = n > 0
            ac = (a * n[sel] + 2) >> 2
            U[sel] = blend(U[sel], yuv[1], ac)
            V[sel] = blend(V[sel], yuv[2], ac)
        return luma, chroma


def blend(src, c, a):
    src = np.asarray(src, np.int64)
    return ((src * (256 - a) + int(c) * a + 128) >> 8).astype(np.uint8)


def pixelate(plane, cov, P):
    """Covered samples of a 2-D plane take their P x P block's rounded mean over its covered samples."""
    h, w = plane.shape
    out = plane.copy()
    if not cov.any():
        return out
    ys, xs = np.nonzero(cov)
    nbx = (w + P - 1) // P
    blk = (ys // P) * nbx + xs // P
    vals = plane[ys, xs].astype(np.int64)
    s = np.bincount(blk, weights=vals, minlength=blk.max() + 1).astype(np.int64)
    n = np.bincount(blk, minlength=blk.max() + 1).astype(np.int64)
    out[ys, xs] = ((s[blk] + n[blk] // 2) // n[blk]).astype(np.uint8)
    return out


def seg_box(seg, r, h, w):
    """A box that holds every pixel a segment can cover (its centre within r): only where the test is evaluated."""
    ax, ay, bx, by = seg
    cl = lambda v, n: int(min(max(v, 0), n))  # noqa: E731
    return (cl(np.floor(min(ax, bx) - r) - 1, w), cl(np.floor(min(ay, by) - r) - 1, h), cl(np.ceil(max(ax, bx) + r) + 1, w),
            cl(np.ceil(max(ay, by) + r) + 1, h))


def segment_covers(xs, ys, seg, r):
    """Pixel centres within r of the segment (ax, ay, bx, by), by the header's float64 steps."""
    ax, ay, bx, by = (float(v) for v in seg)
    cx, cy = xs + 0.5, ys + 0.5
    dx, dy = bx - ax, by - ay
    L2 = dx * dx + dy * dy
    qx, qy = cx - ax, cy - ay
    u = qx * dx + qy * dy
    ex, ey = cx - bx, cy - by
    c = dx * qy - dy * qx
    with np.errstate(divide="ignore", invalid="ignore"):
        mid = c * c / L2
    d2 = np.where(u <= 0, qx * qx + qy * qy, np.where(u >= L2, ex * ex + ey * ey, mid))
    return d2 <= r * r


def text_covers(xs, ys, origin, text, s):
    """Glyph pixels of `text` at origin with scale s (xs, ys inside its cells)."""
    ox, oy = origin
    cx = (xs - ox) // s
    gy = (ys - oy) // s
    ci = cx // 6
    gx = cx - 6 * ci
    codes = np.array([ord(ch) if 0x20 <= ord(ch) <= 0x7E else ord("?") for ch in text], np.int64) - 0x20
    ok = (gx < 5) & (gy < 7)
    g = codes[np.clip(ci, 0, len(codes) - 1)]
    bits = FONT[g, np.clip(gy, 0, 6)].astype(np.int64) >> np.clip(4 - gx, 0, 4) & 1
    return ok & (bits == 1)
