"""The transparent exports (DESIGN 4.19) restated in numpy, shared by the CPU and GPU tiers: straight RGBA / BGRA,
YUVA420P (ffmpeg's yuva420p) and YUVA444P10 (yuva444p10le).

Input: a top-down image c [h][w][4] of the pixels the alpha arithmetic starts from, as alpha_in_np makes it from stored
pixels: under native opacity the stored premultiplied pixels, under any other the stored colour with alpha 255.  The
straight colour of (c, a) is S = a == 0 ? 0 : min(255, (c 255 + a // 2) // a); 4:2:0 chroma takes the block's straight
colour weighted by alpha, min(255, (sum c 255 + sum a // 2) // sum a) (0 when sum a = 0); the 10-bit alpha code is
(a 1023 + 127) // 255."""
import numpy as np

from tests.export_422_np import _coder

FORMATS = ("yuva420p", "yuva444p10")
NAMES = {14: "yuva420p", 15: "yuva444p10"}


def alpha_in_np(frame, native):
    """stored pixels [..., 4] -> what the alpha arithmetic starts from (int64)"""
    c = np.asarray(frame, np.int64).copy()
    if not native:
        c[..., 3] = 255
    return c


def unpremul_np(c, a):
    """the straight channel of stored colour c and alpha a (broadcasting int arrays)"""
    c, a = np.asarray(c, np.int64), np.asarray(a, np.int64)
    return np.where(a == 0, 0, np.minimum(255, (c * 255 + a // 2) // np.maximum(a, 1)))


def straight_np(c):
    """[..., 4] -> the straight pixels [..., 4] (alpha kept)"""
    c = np.asarray(c, np.int64)
    out = c.copy()
    out[..., :3] = unpremul_np(c[..., :3], c[..., 3:4])
    return out


def a10_np(a):
    return (np.asarray(a, np.int64) * 1023 + 127) // 255


def block_straight_np(c):
    """[h][w][4], h and w even -> the alpha-weighted straight colour of every 2x2 block [h / 2][w / 2][3]"""
    h, w = c.shape[:2]
    s = np.asarray(c, np.int64).reshape(h // 2, 2, w // 2, 2, 4).sum(axis=(1, 3))
    sa = s[..., 3:4]
    return np.where(sa == 0, 0, np.minimum(255, (s[..., :3] * 255 + sa // 2) // np.maximum(sa, 1)))


def export_alpha_np(c, fmt, e=0):
    """c as the module docstring says -> straight "rgba" / "bgra" [h][w][4] uint8, or the planes (Y, Cb, Cr, A) of
    "yuva420p" (uint8) / "yuva444p10" (uint16)"""
    c = np.asarray(c, np.int64)
    s = straight_np(c)
    if fmt in ("rgba", "bgra"):
        out = s.astype(np.uint8)
        return out[..., [2, 1, 0, 3]] if fmt == "bgra" else out
    bits = 10 if fmt == "yuva444p10" else 8
    ky, kcb, kcr, yoff, coff, code, dot = _coder(e, bits)
    y = code(dot(ky, s) + (yoff << 16) + (1 << 15), 16)
    if bits == 10:
        m = 4 * s[..., :3]                                  # export_cbcr10_px: a 2x2 block of the pixel
        cb, cr = code(dot(kcb, m) + (coff << 18) + (1 << 17), 18), code(dot(kcr, m) + (coff << 18) + (1 << 17), 18)
        return y.astype(np.uint16), cb.astype(np.uint16), cr.astype(np.uint16), a10_np(c[..., 3]).astype(np.uint16)
    m = block_straight_np(c)
    cb, cr = code(dot(kcb, m) + (coff << 16) + (1 << 15), 16), code(dot(kcr, m) + (coff << 16) + (1 << 15), 16)
    return y.astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8), c[..., 3].astype(np.uint8)


def frame_alpha_np(frame, fmt, e=0, native=True):
    """a read-back frame [h][w][4] (row 0 = bottom) -> what export_frames writes in `fmt` (straight for "rgba" / "bgra")"""
    return export_alpha_np(alpha_in_np(frame[::-1], native), fmt, e)


def scaled_alpha_np(frame, fmt, size, crop=None, e=0, native=True, bg=(0, 0, 0)):
    """a read-back frame -> what export_scaled writes: the area average of the stored channels (native) or of the
    composited pixels (any other opacity, alpha 255), then the alpha arithmetic on that image"""
    from tests.test_export_core import over_np
    from tests.test_export_scaled_core import area_np
    h, w = frame.shape[:2]
    x, y, cw, ch = crop or (0, 0, w, h)
    img = frame[::-1][y:y + ch, x:x + cw].astype(np.int64)
    img = area_np(img if native else over_np(img, bg, False), size)
    return export_alpha_np(img, fmt, e)
