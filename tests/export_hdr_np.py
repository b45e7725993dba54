"""The float64 definition of the BT.2020 HDR exports and overlay (DESIGN 4.22), which tests/test_export_hdr_core.py and the GPU
tests hold export_core.h's float32 code to.  The input is an 8-bit R'G'B' triple (BT.709 primaries, BT.1886 display with
L_B = 0); SDR graphics white sits at 203 cd/m^2 (ITU-R BT.2408), display-referred.  Output: BT.2020 non-constant-luminance
Y'CbCr, limited range, 10 bits, with the PQ (SMPTE ST 2084) or HLG (ITU-R BT.2100, 1000 cd/m^2 display, gamma 1.2) transfer."""
import numpy as np

PQ, HLG = 4, 5                                           # export_core.h's encoding index of EXPORT_PQ / EXPORT_HLG
TRANSFERS = {PQ: "pq", HLG: "hlg"}
WHITE = 203.0                                            # cd/m^2, BT.2408's graphics white

M1, M2 = 2610 / 16384, 2523 / 32
C1, C2, C3 = 3424 / 4096, 2413 / 128, 2392 / 128
HLG_A = 0.17883277
HLG_B = 1 - 4 * HLG_A
HLG_C = 0.5 - HLG_A * np.log(4 * HLG_A)
KR, KG, KB = 0.2627, 0.6780, 0.0593


def _xyz_from(prims, white=(0.3127, 0.3290)):
    P = np.array([[x / y, 1.0, (1 - x - y) / y] for x, y in prims]).T
    W = np.array([white[0] / white[1], 1.0, (1 - white[0] - white[1]) / white[1]])
    return P * np.linalg.solve(P, W)


# BT.709 -> BT.2020 primaries through XYZ, both with D65 white: BT.2087's matrix to 4 decimals
M709_2020 = np.linalg.solve(_xyz_from([(0.708, 0.292), (0.170, 0.797), (0.131, 0.046)]),
                            _xyz_from([(0.64, 0.33), (0.30, 0.60), (0.15, 0.06)]))


def linear(v):
    """BT.1886 with L_B = 0: (v / 255)^2.4 of 8-bit codes"""
    return (np.asarray(v, np.float64) / 255.0) ** 2.4


def pq_oetf(y):
    """ST 2084's inverse EOTF of y = F / 10000"""
    p = np.power(np.maximum(y, 0.0), M1)
    return np.power((C1 + C2 * p) / (1 + C3 * p), M2)


def hlg_oetf(F):
    """BT.2100's inverse OOTF (1000 cd/m^2, gamma 1.2, L_B = 0) and OETF of display light F [..., 3] in cd/m^2"""
    yd = F @ np.array([KR, KG, KB])
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(yd > 0, np.power(np.where(yd > 0, yd, 1.0) / 1000.0, -1.0 / 6.0), 0.0)
    E = F / 1000.0 * s[..., None]
    with np.errstate(invalid="ignore"):
        log = HLG_A * np.log(np.maximum(12 * E - HLG_B, 1e-300)) + HLG_C
    return np.where(E <= 1 / 12, np.sqrt(3 * E), log)


def rgb_prime(c, transfer):
    """E' = (R', G', B') [..., 3] of 8-bit triples c [..., 3]"""
    F = WHITE * linear(c) @ M709_2020.T
    return pq_oetf(F / 10000.0) if transfer == PQ else hlg_oetf(F)


def y_float(e):
    """the unrounded 10-bit Y of E' [..., 3]"""
    return 64 + 876 * (e @ np.array([KR, KG, KB]))


def cbcr_float(e):
    """the unrounded 10-bit (Cb, Cr) [..., 2] of E' [..., 3]"""
    y = e @ np.array([KR, KG, KB])
    return np.stack([512 + 896 * (e[..., 2] - y) / 1.8814, 512 + 896 * (e[..., 0] - y) / 1.4746], -1)


def code(x):
    """rounded half up"""
    return np.floor(np.asarray(x) + 0.5).astype(np.int64)


def unpack(px):
    """uint32 pixels 0xAABBGGRR -> (rgb [..., 3], alpha [...])"""
    px = np.asarray(px, np.uint32)
    return np.stack([px & 255, (px >> 8) & 255, (px >> 16) & 255], -1).astype(np.int64), (px >> 24).astype(np.int64)


def straight(px):
    """export_unpremul of every channel: the straight colour (a == 0: 0), as ints [..., 3]"""
    c, a = unpack(px)
    a3 = a[..., None]
    s = np.where(a3 > 0, (c * 255 + (a3 >> 1)) // np.maximum(a3, 1), 0)
    return np.minimum(s, 255)


def overlay_y_float(px, yd, transfer):
    """the unrounded overlay Y of stored pixels px over the 10-bit codes yd: (a Y_f(S) + (255 - a) Y_D) / 255"""
    _, a = unpack(px)
    yf = y_float(rgb_prime(straight(px), transfer))
    return (a * yf + (255 - a) * np.asarray(yd, np.float64)) / 255.0


def overlay_c_float(pxs, cd, transfer):
    """the unrounded overlay chroma [..., 2] of the n pixels pxs [..., n] of a block over the codes cd [..., 2]:
    512 + sum a_i (C_f(S_i) - 512) / (255 n) + (1 - A / (255 n)) (C_D - 512)"""
    n = np.asarray(pxs).shape[-1]
    _, a = unpack(pxs)
    cf = cbcr_float(rgb_prime(straight(pxs), transfer))
    A = a.sum(-1)
    t = (a[..., None] * (cf - 512)).sum(-2) / (255.0 * n)
    return 512 + t + (1 - A / (255.0 * n))[..., None] * (np.asarray(cd, np.float64) - 512)
