"""The NV12 -> RGB conversion of lwdetr_frame_nv12 (include/lwdetr_b200.h), restated in numpy for the tests.

Integer and exact: u = U - 128, v = V - 128, y' = max(Y - 16, 0) * cY (limited range) or Y * cY (full range),
R = clamp((y' + cRv v + 2^19) >> 20, 0, 255), G = clamp((y' + cGu u + cGv v + 2^19) >> 20, 0, 255),
B = clamp((y' + cBu u + 2^19) >> 20, 0, 255).  Chroma is replicated: pixel (y, x) takes the pair at (y >> 1, x >> 1).
"""
import numpy as np

# colorspace code -> (cY, cRv, cGu, cGv, cBu, limited range)
COEFFS = {
    0: (1220542, 1673527, -409993, -852492, 2116026, True),    # BT.601 limited: OpenCV's 3-decimal table times 2^20
    1: (1220945, 1879825, -223607, -558796, 2215014, True),    # BT.709 limited
    2: (1048576, 1470104, -360853, -748826, 1858077, False),   # BT.601 full
    3: (1048576, 1651297, -196424, -490864, 1945738, False),   # BT.709 full
}
NAMES = {"bt601": 0, "bt709": 1, "bt601_full": 2, "bt709_full": 3}
KR_KB = {0: (0.299, 0.114), 1: (0.2126, 0.0722), 2: (0.299, 0.114), 3: (0.2126, 0.0722)}


def code(colorspace):
    return NAMES[colorspace] if isinstance(colorspace, str) else int(colorspace)


def exact_coeffs(colorspace):
    """(cY, cRv, cGu, cGv, cBu) as real numbers from (Kr, Kb), with 255/219 luma and 255/224 chroma scaling when limited."""
    cs = code(colorspace)
    kr, kb = KR_KB[cs]
    kg = 1.0 - kr - kb
    ys, cs_ = (255 / 219, 255 / 224) if COEFFS[cs][5] else (1.0, 1.0)
    return (ys, 2 * (1 - kr) * cs_, -2 * kb * (1 - kb) / kg * cs_, -2 * kr * (1 - kr) / kg * cs_, 2 * (1 - kb) * cs_)


def yuv_to_rgb(Y, U, V, colorspace):
    """Per-pixel conversion of equally shaped uint8 arrays Y, U, V -> uint8 [..., 3]."""
    cY, cRv, cGu, cGv, cBu, limited = COEFFS[code(colorspace)]
    Y, u, v = (np.asarray(a, dtype=np.int32) for a in (Y, U, V))
    u, v = u - 128, v - 128
    yp = (np.maximum(Y - 16, 0) if limited else Y) * cY
    half = 1 << 19
    out = np.stack([yp + cRv * v + half, yp + cGu * u + cGv * v + half, yp + cBu * u + half], axis=-1) >> 20
    return np.clip(out, 0, 255).astype(np.uint8)


def yuv_to_rgb_float(Y, U, V, colorspace):
    """The same conversion in float64 with the exact coefficients, rounded half up: the yardstick of the integer rows."""
    cY, cRv, cGu, cGv, cBu = exact_coeffs(colorspace)
    Y, u, v = (np.asarray(a, dtype=np.float64) for a in (Y, U, V))
    u, v = u - 128, v - 128
    yp = (np.maximum(Y - 16, 0) if COEFFS[code(colorspace)][5] else Y) * cY
    out = np.floor(np.stack([yp + cRv * v, yp + cGu * u + cGv * v, yp + cBu * u], axis=-1) + 0.5)
    return np.clip(out, 0, 255).astype(np.uint8)


def nv12_to_rgb(luma, chroma, colorspace):
    """luma uint8 [h, w], chroma uint8 [ceil(h/2), 2 * ceil(w/2)] (U, V pairs) -> RGB uint8 [h, w, 3]."""
    luma, chroma = np.asarray(luma), np.asarray(chroma)
    h, w = luma.shape
    assert chroma.shape == ((h + 1) // 2, 2 * ((w + 1) // 2)), (luma.shape, chroma.shape)
    U = np.repeat(np.repeat(chroma[:, 0::2], 2, axis=0), 2, axis=1)[:h, :w]
    V = np.repeat(np.repeat(chroma[:, 1::2], 2, axis=0), 2, axis=1)[:h, :w]
    return yuv_to_rgb(luma, U, V, colorspace)


def split_packed(nv12):
    """A packed NV12 frame [3h/2, w] (h, w even) -> (luma [h, w], chroma [h/2, w]) views."""
    rows = nv12.shape[0]
    h = rows * 2 // 3
    return nv12[:h], nv12[h:]
