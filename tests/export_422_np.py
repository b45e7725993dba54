"""The 4:2:2 export and overlay (DESIGN 4.18) restated in numpy, shared by the CPU and GPU tiers.

Export: a composited top-down image c [h][w][>= 3] -> YUV422P / YUV422P10 (Y [h, w], Cb and Cr [h, w / 2]) or UYVY
([h, 2 w] bytes, Cb Y0 Cr Y1 per pixel pair).  The chroma of a pixel pair (c0, c1) is the 4:2:0 chroma of the block whose
two rows are that pair: 8 bits from the byte average (2 a + 2 b + 2) >> 2, 10 bits from the exact sums 2 (a + b).

Overlay: what one entry leaves in its rectangle's planes, from the read-back frame and the planes before the call, as
tests/overlay_planes_np.py states it for the other formats; UYVY is blended as YUV422P's planes and packed again."""
import numpy as np

from tests.overlay_planes_np import cbcr8_np, cbcr10_np, y_np
from tests.test_export_matrix_core import coef_py

FORMATS = ("yuv422p", "yuv422p10", "uyvy")
NAMES = {10: "yuv422p", 11: "yuv422p10", 12: "uyvy"}
CODES = {v: k for k, v in NAMES.items()}


def _coder(e, bits):
    ky, kcb, kcr, yoff, coff, top, full = coef_py(e, bits)
    code = (lambda acc, sh: np.minimum(acc >> sh, top)) if full else (lambda acc, sh: acc >> sh)
    dot = lambda k, v: k[0] * v[..., 0] + k[1] * v[..., 1] + k[2] * v[..., 2]
    return ky, kcb, kcr, yoff, coff, code, dot


def pair_sums(c):
    """the per-channel sums of the 2x2 blocks whose two rows are each pixel pair: 2 (c0 + c1), [h, w / 2, channels]"""
    c = np.asarray(c, np.int64)
    h, w = c.shape[:2]
    return 2 * c.reshape(h, w // 2, 2, -1).sum(axis=2)


def export422_np(c, fmt, e):
    c = np.asarray(c, np.int64)
    bits = 10 if fmt == "yuv422p10" else 8
    ky, kcb, kcr, yoff, coff, code, dot = _coder(e, bits)
    y = code(dot(ky, c) + (yoff << 16) + (1 << 15), 16)
    s = pair_sums(c[..., :3])
    if bits == 10:
        cb, cr = code(dot(kcb, s) + (coff << 18) + (1 << 17), 18), code(dot(kcr, s) + (coff << 18) + (1 << 17), 18)
        return y.astype(np.uint16), cb.astype(np.uint16), cr.astype(np.uint16)
    m = (s + 2) >> 2
    cb, cr = code(dot(kcb, m) + (coff << 16) + (1 << 15), 16), code(dot(kcr, m) + (coff << 16) + (1 << 15), 16)
    y, cb, cr = y.astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8)
    return uyvy_of(y, cb, cr) if fmt == "uyvy" else (y, cb, cr)


def uyvy_of(y, cb, cr):
    """planar 4:2:2 bytes packed as UYVY: [..., h, 2 w]"""
    out = np.empty(y.shape[:-1] + (2 * y.shape[-1],), np.uint8)
    out[..., 0::4], out[..., 1::2], out[..., 2::4] = cb, y, cr
    return out


def planar_of(u):
    """UYVY bytes [..., h, 2 w] -> (Y, Cb, Cr)"""
    return u[..., 1::2], u[..., 0::4], u[..., 2::4]


def overlay422_np(frame, planes, fmt, e, native):
    """frame: read-back [h][w][4] (row 0 = bottom); planes: the rectangle's planes before the call ((Y, Cb, Cr), or (UYVY,))
    -> the planes after.  Native opacity blends, leaving samples no non-zero pixel (pair) covers as they were, all 16 bits
    of a 10-bit sample included; any other opacity is the export."""
    c = frame[::-1].astype(np.int64)
    h, w = c.shape[:2]
    if not native:
        c[..., 3] = 255
    nz = (c != 0).any(axis=-1) if native else np.ones((h, w), bool)
    pnz = nz.reshape(h, w // 2, 2).any(axis=-1)
    src = planar_of(planes[0]) if fmt == "uyvy" else planes
    yb, cbd, crd = (p.astype(np.int64) for p in src)
    s = pair_sums(c)
    if fmt == "yuv422p10":
        y = y_np(e, 10, c, yb & 1023)
        cb, cr = cbcr10_np(e, s, cbd & 1023, crd & 1023)
    else:
        y = y_np(e, 8, c, yb)
        cb, cr = cbcr8_np(e, (s + 2) >> 2, cbd, crd)
    dt = np.uint16 if fmt == "yuv422p10" else np.uint8
    y = np.where(nz, y, yb).astype(dt)
    cb, cr = np.where(pnz, cb, cbd).astype(dt), np.where(pnz, cr, crd).astype(dt)
    return [uyvy_of(y, cb, cr)] if fmt == "uyvy" else [y, cb, cr]
