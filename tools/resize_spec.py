"""The resize that `forward_frames` performs on the device, restated on the CPU  --  TEST INFRASTRUCTURE ONLY.

The separable triangle filter of PIL.Image.resize(BILINEAR) and F.interpolate(mode="bilinear", antialias=True), as
csrc/resize.cu and include/lwdetr_b200.h (lwdetr_frame) state it.  Per axis n_in -> n_out: scale = n_in / n_out,
support = max(scale, 1); output o has centre c = (o + 0.5) * scale, taps x in [max(int(c - support + 0.5), 0),
min(int(c + support + 0.5), n_in)), weight max(0, 1 - |x - c + 0.5| / support) over the sum of the weights.  Horizontal
pass, then vertical; the result is rounded half up (floor(v + 0.5) in fp32) to an integer level and clamped to [0, 255].

Tap ranges and weights are computed in fp32, operation by operation as the kernel does.  The two passes' sums are taken in
float64 and stored as fp32 (the kernel keeps the row pass in fp32 too): the restatement then carries no summation-order
noise of its own, and a kernel that sums in fp32 in any order lands within ~1e-4 levels of it.
"""
import numpy as np

_f = np.float32


def axis_weights(n_in, n_out):
    """Dense [n_out, n_in] fp32 matrix of the normalised tap weights of one axis."""
    scale = _f(n_in) / _f(n_out)
    support = max(scale, _f(1.0))
    centre = (np.arange(n_out, dtype=np.float32) + _f(0.5)) * scale
    lo = np.maximum((centre - support + _f(0.5)).astype(np.int32), 0)
    hi = np.minimum((centre + support + _f(0.5)).astype(np.int32), n_in)
    m = np.zeros((n_out, n_in), dtype=np.float32)
    for o in range(n_out):
        x = np.arange(lo[o], hi[o], dtype=np.int32).astype(np.float32)
        w = np.maximum(_f(0.0), _f(1.0) - np.abs(x - centre[o] + _f(0.5)) / support)
        m[o, lo[o]:hi[o]] = w / np.cumsum(w, dtype=np.float32)[-1]          # sequential fp32 sum, as the kernel
    return m


def resize_levels(frame, dst_h, dst_w):
    """uint8 (or float) [h, w, C] -> fp32 [dst_h, dst_w, C] in levels, BEFORE rounding."""
    img = np.asarray(frame)
    h, w = img.shape[:2]
    rows = np.einsum("ox,yxc->yoc", axis_weights(w, dst_w).astype(np.float64), img.astype(np.float64), optimize=True).astype(np.float32)
    return np.einsum("oy,yxc->oxc", axis_weights(h, dst_h).astype(np.float64), rows.astype(np.float64), optimize=True).astype(np.float32)


def round_levels(levels):
    """Round half up to an integer level and clamp: fp32 levels -> uint8."""
    return np.clip(np.floor(levels.astype(np.float32) + _f(0.5)), 0, 255).astype(np.uint8)


def resize_u8(frame, dst_h, dst_w):
    """uint8 [h, w, 3] -> uint8 [dst_h, dst_w, 3]: the image a host resize would hand to the uint8 input path."""
    return round_levels(resize_levels(frame, dst_h, dst_w))


def tie_pixels(levels, eps=1e-3):
    """Boolean map of values whose fractional part lies within eps of one half: a summation-order difference may round them
    to either neighbouring level."""
    lv = levels.astype(np.float64)
    return np.abs(lv - np.floor(lv) - 0.5) <= eps


def normalise(u8, mean, std):
    """(x / 255 - mean) / std in fp32 with IEEE divisions (ToTensor, Normalize): uint8 [..., 3] -> fp32 [..., 3]."""
    return (u8.astype(np.float32) / _f(255.0) - np.asarray(mean, dtype=np.float32)) / np.asarray(std, dtype=np.float32)


def canvas(frames, dsts, size, mean, std):
    """What the device path presents to the patch embedding: each frame resized to its (dst_h, dst_w), normalised, top-left
    on a zero [H, W] canvas.  Returns (fp32 [B, H, W, 3], uint8 resized-and-zero-padded [B, H, W, 3], bool mask [B, H, W])."""
    H, W = size
    out = np.zeros((len(frames), H, W, 3), dtype=np.float32)
    u8 = np.zeros((len(frames), H, W, 3), dtype=np.uint8)
    mask = np.ones((len(frames), H, W), dtype=bool)
    for b, (fr, (dh, dw)) in enumerate(zip(frames, dsts)):
        r = resize_u8(fr, dh, dw)
        u8[b, :dh, :dw] = r
        out[b, :dh, :dw] = normalise(r, mean, std)
        mask[b, :dh, :dw] = False
    return out, u8, mask
