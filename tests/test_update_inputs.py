"""What the eight ways into an update do with their arguments, without a GPU: capi.cu built against the fake runtime of
tests/fakecuda.  For every entry point and every kind of bad or unusual input (null handle, PCM, mask or right channel;
wrong bsz; misaligned device pointers; masks that are all zero, all one or uneven, with and without keyframe
interpolation; a renderer a failed rebuild left unbuilt; two of these at once), the return code, the error text and the
number of kernels launched are pinned.  A refused call launches nothing."""
import ctypes as C

import numpy as np
import pytest

from tests import fakecuda
from tests.test_handle_lifetime import BATCH, Fake

OK, EINVAL, ECUDA = 0, -1, -3
N = 1024
CONFIG = {
    "bars": ("bars", dict(n=N, w=64, h=32)),
    "wave": ("wave", dict(n=N, w=64, h=32)),
    "interp": ("bars", dict(n=N, w=64, h=32, transform_smooth=1, interpolate=1, ur=30.0, fr=60.0)),
}
PCM = ("update", "update_masked", "update_device", "update_device_masked", "update_device_after")
DEVICE = ("update_device", "update_device_masked", "update_device_after")
MASKED = ("update_masked", "update_device_masked", "update_rings_masked")
ENTRIES = PCM + ("update_rings", "update_rings_masked", "raster_textures")
UNEVEN, ALL, NONE = [1, 0], [1, 1], [0, 0]

# case: (configuration, entry points, input changes, unbuilt renderer)
#   input changes: handle / l / r / mask = None, l / r = "+4" (misaligned by 4 bytes), bsz, modified, mask = [bytes]
CASES = {
    "plain": ("bars", ENTRIES, {}, False),
    "silent": ("bars", ("update", "update_device", "update_device_after", "update_rings"), dict(modified=0), False),
    "null_handle": ("bars", ENTRIES, dict(handle=None), False),
    "null_pcm": ("bars", PCM + ("raster_textures",), dict(l=None), False),
    "null_mask": ("bars", MASKED, dict(mask=None), False),
    "null_rb_bars": ("bars", PCM + ("raster_textures",), dict(r=None), False),
    "null_rb_bars_silent": ("bars", PCM, dict(r=None, modified=0, mask=NONE), False),
    "null_rb_wave": ("wave", PCM + ("raster_textures",), dict(r=None), False),
    "wrong_bsz": ("bars", PCM, dict(bsz=N - 1), False),
    "misaligned_l": ("bars", PCM, dict(l="+4"), False),
    "misaligned_r": ("bars", PCM, dict(r="+4"), False),
    "mask_all_zero": ("bars", MASKED, dict(mask=NONE), False),
    "mask_all_one": ("bars", MASKED, dict(mask=ALL), False),
    "mask_uneven": ("bars", MASKED, dict(mask=UNEVEN), False),
    "mask_all_one_interp": ("interp", MASKED, dict(mask=ALL), False),
    "mask_uneven_interp": ("interp", MASKED, dict(mask=UNEVEN), False),
    "unbuilt": ("bars", ENTRIES, {}, True),
    "unbuilt_silent": ("bars", ("update", "update_device", "update_device_after", "update_rings"), dict(modified=0), True),
    "unbuilt_wrong_bsz": ("bars", PCM, dict(bsz=N - 1), True),
    "unbuilt_null_rb": ("bars", PCM, dict(r=None), True),
    "unbuilt_mask_uneven_interp": ("interp", MASKED, dict(mask=UNEVEN), True),
}

NULL = "null argument"
ALIGN = "device PCM pointers must be 16-byte aligned"
UNBUILT = "a reconfigure or resize failed"
MASKREF = "per-stream modified masks are not available with keyframe interpolation"


def bsz(entry):
    return f"glava_b200_{entry}: bsz {N - 1} != setbufsize {N}"


def rb(entry, name):
    return f"glava_b200_{entry}: module 'bars' reads both channels, {name} is null"


# (case, entry point): (return code, error text it contains, kernels launched)
EXPECT = {
    **{("plain", e): (OK, None, 2) for e in ENTRIES if e != "raster_textures"},
    ("plain", "raster_textures"): (OK, None, 1),
    **{("silent", e): (OK, None, 1) for e in CASES["silent"][1]},
    **{("null_handle", e): (EINVAL, NULL, 0) for e in ENTRIES},
    **{("null_pcm", e): (EINVAL, f"glava_b200_{e}: {NULL}", 0) for e in PCM + ("raster_textures",)},
    **{("null_mask", e): (EINVAL, f"glava_b200_{e}: {NULL}", 0) for e in MASKED},
    ("null_rb_bars", "update"): (EINVAL, rb("update", "rb"), 0),
    ("null_rb_bars", "update_masked"): (EINVAL, rb("update_masked", "rb"), 0),
    ("null_rb_bars", "update_device"): (EINVAL, rb("update_device", "d_rb"), 0),
    ("null_rb_bars", "update_device_masked"): (EINVAL, rb("update_device_masked", "d_rb"), 0),
    ("null_rb_bars", "update_device_after"): (EINVAL, rb("update_device_after", "d_rb"), 0),
    ("null_rb_bars", "raster_textures"): (OK, None, 1),
    # an unmodified update does not read rb, but a device-pointer masked update wants d_rb for any mask
    ("null_rb_bars_silent", "update"): (OK, None, 1),
    ("null_rb_bars_silent", "update_masked"): (OK, None, 1),
    ("null_rb_bars_silent", "update_device"): (OK, None, 1),
    ("null_rb_bars_silent", "update_device_masked"): (EINVAL, rb("update_device_masked", "d_rb"), 0),
    ("null_rb_bars_silent", "update_device_after"): (OK, None, 1),
    **{("null_rb_wave", e): (OK, None, 2) for e in PCM},
    ("null_rb_wave", "raster_textures"): (OK, None, 1),
    **{("wrong_bsz", e): (EINVAL, bsz(e), 0) for e in PCM},
    **{("misaligned_l", e): (OK, None, 2) for e in ("update", "update_masked")},
    **{("misaligned_l", e): (EINVAL, ALIGN, 0) for e in DEVICE},
    **{("misaligned_r", e): (OK, None, 2) for e in ("update", "update_masked")},
    **{("misaligned_r", e): (EINVAL, ALIGN, 0) for e in DEVICE},
    **{("mask_all_zero", e): (OK, None, 1) for e in MASKED},
    **{("mask_all_one", e): (OK, None, 2) for e in MASKED},
    **{("mask_uneven", e): (OK, None, 2) for e in MASKED},
    **{("mask_all_one_interp", e): (OK, None, 5) for e in MASKED},
    **{("mask_uneven_interp", e): (EINVAL, MASKREF, 0) for e in MASKED},
    **{("unbuilt", e): (ECUDA, UNBUILT, 0) for e in ENTRIES},
    **{("unbuilt_silent", e): (ECUDA, UNBUILT, 0) for e in CASES["unbuilt_silent"][1]},
    **{("unbuilt_wrong_bsz", e): (EINVAL, bsz(e), 0) for e in PCM},
    ("unbuilt_null_rb", "update"): (EINVAL, rb("update", "rb"), 0),
    ("unbuilt_null_rb", "update_masked"): (EINVAL, rb("update_masked", "rb"), 0),
    ("unbuilt_null_rb", "update_device"): (EINVAL, rb("update_device", "d_rb"), 0),
    ("unbuilt_null_rb", "update_device_masked"): (EINVAL, rb("update_device_masked", "d_rb"), 0),
    ("unbuilt_null_rb", "update_device_after"): (EINVAL, rb("update_device_after", "d_rb"), 0),
    # the host path reports the unbuilt renderer first, the device and ring paths the mask
    ("unbuilt_mask_uneven_interp", "update_masked"): (ECUDA, UNBUILT, 0),
    ("unbuilt_mask_uneven_interp", "update_device_masked"): (EINVAL, MASKREF, 0),
    ("unbuilt_mask_uneven_interp", "update_rings_masked"): (EINVAL, MASKREF, 0),
}


@pytest.fixture(scope="module")
def fake():
    if fakecuda.cuda_include() is None:
        pytest.skip("no CUDA toolkit headers")
    return Fake()


def call(fake, case, entry):
    """run one entry point on a fresh renderer; returns (rc, last error, kernels launched by the call)"""
    cfg, _, change, unbuilt = CASES[case]
    module, kw = CONFIG[cfg]
    L = fake.L
    L.fake_fail_at(-1)
    p = fake.params(module, **kw)
    h = fake.new(p)
    assert h
    try:
        if unbuilt:
            q = fake.params(module, **kw)
            q.smooth_factor = 0.02 if p.smooth_factor != 0.02 else 0.03
            L.fake_fail_at(0)
            assert L.glava_b200_reconfigure(h, C.byref(q)) != 0
            L.fake_fail_at(-1)
        pcm = np.zeros((2 * BATCH * N + 16,), np.float32)
        base = pcm.ctypes.data + (-pcm.ctypes.data) % 64
        ptr = {"l": base, "r": base + BATCH * N * 4}
        for k in ("l", "r"):
            if k in change:
                ptr[k] = None if change[k] is None else ptr[k] + 4
        mask = change.get("mask", ALL)
        m = None if mask is None else np.array(mask, np.uint8)
        mp = None if m is None else m.ctypes.data
        n, mod = change.get("bsz", N), change.get("modified", 1)
        handle = change.get("handle", h)
        ready = L.glava_b200_input_event(h)
        tex = np.zeros((BATCH, N), np.uint16)
        tl = None if ptr["l"] is None else tex.ctypes.data
        tr = None if ptr["r"] is None else tex.ctypes.data
        before = L.fake_launches()
        rc = {
            "update": lambda: L.glava_b200_update(handle, ptr["l"], ptr["r"], n, mod),
            "update_masked": lambda: L.glava_b200_update_masked(handle, ptr["l"], ptr["r"], n, mp),
            "update_device": lambda: L.glava_b200_update_device(handle, ptr["l"], ptr["r"], n, mod),
            "update_device_masked": lambda: L.glava_b200_update_device_masked(handle, ptr["l"], ptr["r"], n, mp),
            "update_device_after": lambda: L.glava_b200_update_device_after(handle, ptr["l"], ptr["r"], n, mod, ready),
            "update_rings": lambda: L.glava_b200_update_rings(handle, mod),
            "update_rings_masked": lambda: L.glava_b200_update_rings_masked(handle, mp),
            "raster_textures": lambda: L.glava_b200_raster_textures(handle, tl, tr),
        }[entry]()
        return rc, L.glava_b200_last_error().decode(), L.fake_launches() - before
    finally:
        L.glava_b200_destroy(h)


@pytest.mark.parametrize("case,entry", sorted(EXPECT))
def test_update_input(fake, case, entry):
    assert entry in CASES[case][1]
    want_rc, want_text, want_launches = EXPECT[(case, entry)]
    rc, text, launches = call(fake, case, entry)
    assert rc == want_rc, text
    if want_text is not None:
        assert want_text in text
    assert launches == want_launches


def test_every_case_has_an_expectation():
    assert sorted(EXPECT) == sorted((c, e) for c, (_, entries, _, _) in CASES.items() for e in entries)
