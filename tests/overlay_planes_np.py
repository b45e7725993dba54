"""The overlay onto decoded pictures (glava_b200_overlay_planes, DESIGN 4.17) restated in numpy: what one entry leaves in the
planes of its rectangle, from the read-back frame and the planes' samples before the call.  Shared by the CPU and GPU tiers.

Planes are numpy arrays of samples covering the rectangle: Y [h, w]; NV12 CbCr [h / 2, w] bytes, P010 CbCr [h / 2, w]
uint16 (Cb, Cr interleaved); I420 / YUV420P10 Cb and Cr [h / 2, w / 2]; YUV444 / YUV444P10 Cb and Cr [h, w]."""
import numpy as np

from tests.test_export_matrix_core import coef_py

FORMATS = ("nv12", "i420", "yuv444", "p010", "yuv420p10", "yuv444p10")
WIDE = ("p010", "yuv420p10", "yuv444p10")
C420 = ("nv12", "i420", "p010", "yuv420p10")


def code_of(v, fmt):
    """the 10-bit code a sample holds"""
    v = v.astype(np.int64)
    return v >> 6 if fmt == "p010" else v & 1023


def sample_of(code, fmt):
    return code << 6 if fmt == "p010" else code


def y_np(e, bits, c, vd):
    """Y codes of pixels c [..., 4] (stored, premultiplied) over codes vd"""
    ky, _, _, yoff, _, top, _ = coef_py(e, bits)
    a = c[..., 3]
    t = yoff * a + (255 - a) * vd
    frac = (t * 65536 + 127) // 255
    dot = ky[0] * c[..., 0] + ky[1] * c[..., 1] + ky[2] * c[..., 2]
    return np.clip((dot + frac + (1 << 15)) >> 16, 0, top)


def cbcr8_np(e, m, cbd, crd):
    """8-bit (Cb, Cr) of block averages m [..., 4] (alpha included) over codes cbd, crd"""
    _, kcb, kcr, _, coff, _, _ = coef_py(e, 8)
    a = m[..., 3]
    frac = lambda vd: ((coff * a + (255 - a) * vd) * 65536 + 127) // 255
    dot = lambda k: k[0] * m[..., 0] + k[1] * m[..., 1] + k[2] * m[..., 2]
    return (np.clip((dot(kcb) + frac(cbd) + (1 << 15)) >> 16, 0, 255), np.clip((dot(kcr) + frac(crd) + (1 << 15)) >> 16, 0, 255))


def cbcr10_np(e, s, cbd, crd):
    """10-bit (Cb, Cr) of block sums s [..., 4] (0..1020 per channel, alpha included) over codes cbd, crd"""
    _, kcb, kcr, _, coff, _, _ = coef_py(e, 10)
    sa = s[..., 3]
    g = lambda vd: ((coff * sa + (1020 - sa) * vd) * 65536 + 509) // 1020
    dot = lambda k: k[0] * s[..., 0] + k[1] * s[..., 1] + k[2] * s[..., 2]
    return (np.clip((dot(kcb) + 4 * g(cbd) + (1 << 17)) >> 18, 0, 1023), np.clip((dot(kcr) + 4 * g(crd) + (1 << 17)) >> 18, 0, 1023))


def planes_np(frame, planes, fmt, e, native):
    """frame: read-back [h][w][4] (row 0 = bottom); planes: the rectangle's planes before the call -> the planes after.
    Native opacity blends, leaving samples that no non-zero pixel covers as they were; any other opacity is the export
    (the blend of every pixel at alpha 255, which gives export_frames' codes)."""
    c = frame[::-1].astype(np.int64)
    h, w = c.shape[:2]
    if not native:
        c[..., 3] = 255
    nz = (c != 0).any(axis=-1) if native else np.ones((h, w), bool)
    wide = fmt in WIDE
    out = [p.copy() for p in planes]
    yb = planes[0].astype(np.int64)
    if wide:
        y = sample_of(y_np(e, 10, c, code_of(yb, fmt)), fmt)
    else:
        y = y_np(e, 8, c, yb)
    out[0] = np.where(nz, y, yb).astype(planes[0].dtype)
    if fmt in C420:
        blocks = c.reshape(h // 2, 2, w // 2, 2, 4).sum(axis=(1, 3))
        bnz = nz.reshape(h // 2, 2, w // 2, 2).any(axis=(1, 3))
    else:
        blocks, bnz = c, nz
    if fmt in ("nv12", "p010"):
        uv = planes[1].astype(np.int64).reshape(h // 2, w // 2, 2)
        cbd, crd = uv[..., 0], uv[..., 1]
    else:
        cbd, crd = planes[1].astype(np.int64), planes[2].astype(np.int64)
    if wide:
        s = blocks if fmt in C420 else 4 * blocks
        cb, cr = cbcr10_np(e, s, code_of(cbd, fmt), code_of(crd, fmt))
        cb, cr = sample_of(cb, fmt), sample_of(cr, fmt)
    else:
        m = (blocks + 2) >> 2 if fmt in C420 else blocks
        cb, cr = cbcr8_np(e, m, cbd, crd)
    cb, cr = np.where(bnz, cb, cbd), np.where(bnz, cr, crd)
    if fmt in ("nv12", "p010"):
        out[1] = np.stack([cb, cr], axis=-1).reshape(h // 2, w).astype(planes[1].dtype)
    else:
        out[1], out[2] = cb.astype(planes[1].dtype), cr.astype(planes[2].dtype)
    return out
