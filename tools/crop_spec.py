"""The detection crops of lwdetr_crops (include/lwdetr_b200.h), restated in numpy  --  TEST INFRASTRUCTURE ONLY.

Crop rectangle: cx0 = clamp(floor(x1), 0, w), cx1 = clamp(floor(x2), 0, w), rows likewise; valid when cx1 > cx0, cy1 > cy0 and
every coordinate is finite.  Two filters, per axis n_in -> n_out with scale = n_in / n_out in fp32:
  "bilinear" (cv2.resize INTER_LINEAR): f = (o + 0.5) * scale - 0.5, s = floor(f), t = f - s; s < 0: s = 0, t = 0;
    s >= n_in - 1: the one tap n_in - 1; else taps s, s + 1 with weights 1 - t, t;
  "antialias": resize_spec's triangle filter (any downscale).
Tap weights are fp32, computed operation by operation as the kernel does; the two passes' sums are float64 stored as fp32
(as resize_spec), then rounded half up to a level and clamped.  Values: resize_spec.normalise of the levels, or the levels.
NV12: the frame converted by yuv_spec (chroma of the whole frame), then the RGB rule.
"""
import numpy as np

import resize_spec
import yuv_spec

_f = np.float32
FILTERS = ("bilinear", "antialias")


def crop_rect(box, h, w):
    """(cx0, cy0, cx1, cy1) of an xyxy box in an h x w frame, or None when the crop is invalid."""
    b = np.asarray(box, dtype=np.float32)
    if not np.all(np.isfinite(b)):
        return None
    x0, x1 = (int(min(max(np.floor(v), 0.0), w)) for v in (b[0], b[2]))
    y0, y1 = (int(min(max(np.floor(v), 0.0), h)) for v in (b[1], b[3]))
    return (x0, y0, x1, y1) if x1 > x0 and y1 > y0 else None


def bilinear_weights(n_in, n_out):
    """Dense [n_out, n_in] fp32 matrix of cv2 INTER_LINEAR's taps as the contract states them (float weights)."""
    scale = _f(n_in) / _f(n_out)
    m = np.zeros((n_out, n_in), dtype=np.float32)
    for o in range(n_out):
        f = (_f(o) + _f(0.5)) * scale - _f(0.5)
        s = int(np.floor(f))
        t = f - _f(np.floor(f))
        if s < 0:
            s, t = 0, _f(0.0)
        if s >= n_in - 1:
            m[o, n_in - 1] = 1.0
        else:
            m[o, s] = _f(1.0) - t
            m[o, s + 1] += t
    return m


def axis_weights(filter, n_in, n_out):
    if filter == "bilinear":
        return bilinear_weights(n_in, n_out)
    if filter == "antialias":
        return resize_spec.axis_weights(n_in, n_out)
    raise ValueError(filter)


def resize_levels(img, dst_h, dst_w, filter):
    """uint8 [h, w, 3] -> fp32 [dst_h, dst_w, 3] levels before rounding (float64 pass sums, each pass stored as fp32)."""
    h, w = img.shape[:2]
    rows = np.einsum("ox,yxc->yoc", axis_weights(filter, w, dst_w).astype(np.float64), img.astype(np.float64), optimize=True).astype(np.float32)
    return np.einsum("oy,yxc->oxc", axis_weights(filter, h, dst_h).astype(np.float64), rows.astype(np.float64), optimize=True).astype(np.float32)


def crop_levels(frame, box, size, filter):
    """fp32 [h, w, 3] levels before rounding of one box of an RGB uint8 [H, W, 3] frame, or None for an invalid crop."""
    r = crop_rect(box, frame.shape[0], frame.shape[1])
    if r is None:
        return None
    x0, y0, x1, y1 = r
    return resize_levels(frame[y0:y1, x0:x1], size[0], size[1], filter)


def crops(frames, boxes, frame_index, size, filter, mean=None, std=None, normalize=True):
    """RGB uint8 frames (list of [H, W, 3]) -> (values fp32 [N, 3, h, w], levels uint8 [N, 3, h, w], levels before rounding
    fp32 [N, 3, h, w], valid bool [N]).  Invalid crops are zeros."""
    N = len(boxes)
    h, w = size
    vals = np.zeros((N, 3, h, w), np.float32)
    u8 = np.zeros((N, 3, h, w), np.uint8)
    raw = np.zeros((N, 3, h, w), np.float32)
    valid = np.zeros(N, bool)
    for i, (box, f) in enumerate(zip(boxes, frame_index)):
        if not 0 <= f < len(frames):
            continue
        lv = crop_levels(frames[f], box, size, filter)
        if lv is None:
            continue
        valid[i] = True
        q = resize_spec.round_levels(lv)
        raw[i] = lv.transpose(2, 0, 1)
        u8[i] = q.transpose(2, 0, 1)
        vals[i] = (resize_spec.normalise(q, mean, std) if normalize else q.astype(np.float32)).transpose(2, 0, 1)
    return vals, u8, raw, valid


def nv12_frames(pairs, colorspaces):
    """(luma, chroma) uint8 pairs -> the RGB frames the NV12 crops are taken from."""
    return [yuv_spec.nv12_to_rgb(y, c, cs) for (y, c), cs in zip(pairs, colorspaces)]


def select(scores, boxes, sizes, threshold):
    """lwdetr_crop_select: (frame, flat entry, box) of every entry with score > threshold (fp32) and a valid crop, in (frame,
    entry) order."""
    scores = np.asarray(scores, np.float32)
    B, k = scores.shape
    out = []
    for b in range(B):
        for j in range(k):
            if scores[b, j] > _f(threshold) and crop_rect(boxes[b][j], *sizes[b]) is not None:
                out.append((b, b * k + j, np.asarray(boxes[b][j], np.float32)))
    return out
