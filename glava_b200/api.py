"""ctypes binding of include/glava_b200.h."""
import ctypes as C
import os

import numpy as np

MODULES = ("bars", "radial", "circle", "graph", "wave", "test")
_HERE = os.path.dirname(os.path.abspath(__file__))


class GlavaError(RuntimeError):
    pass


class Color(C.Structure):
    _fields_ = [("mode", C.c_int), ("lo", C.c_float * 4), ("hi", C.c_float * 4), ("gradient", C.c_float)]


class ColorOp(C.Structure):
    _fields_ = [("op", C.c_uint8), ("dst", C.c_uint8), ("a", C.c_uint8), ("b", C.c_uint8), ("imm", C.c_float)]


class ColorProg(C.Structure):
    """glava_b200_color_prog: a compiled colour expression (mode 2 of the colour it belongs to)"""
    _fields_ = [("n_ops", C.c_int), ("result", C.c_int), ("ops", ColorOp * 64)]


class Params(C.Structure):
    """struct glava_b200_params (include/glava_b200.h) — same field order."""
    _fields_ = [
        ("n", C.c_int), ("fft_scale", C.c_float), ("fft_cutoff", C.c_float), ("gravity_step", C.c_float),
        ("ur", C.c_float), ("avg_frames", C.c_int), ("avg_window", C.c_int), ("accel_fft", C.c_int),
        ("smooth_pass", C.c_int), ("smooth_factor", C.c_float), ("sample_range", C.c_float),
        ("sample_scale", C.c_float), ("hybrid_weight", C.c_float), ("sample_mode", C.c_int),
        ("round_formula", C.c_int),
        ("module", C.c_int), ("w", C.c_int), ("h", C.c_int), ("channels", C.c_int), ("premultiply_alpha", C.c_int),
        ("bars_width", C.c_float), ("bars_gap", C.c_float), ("bars_outline_width", C.c_float), ("bars_amplify", C.c_float),
        ("bars_color", Color), ("bars_outline_mode", C.c_int), ("bars_outline", C.c_float * 4),
        ("bars_direction", C.c_int), ("bars_invert", C.c_int), ("bars_flip", C.c_int), ("bars_mirror_yx", C.c_int),
        ("radial_radius", C.c_float), ("radial_line", C.c_float), ("radial_line_half", C.c_float),
        ("radial_outline", C.c_float * 4), ("radial_nbars", C.c_int), ("radial_bar_width", C.c_float),
        ("radial_amplify", C.c_float), ("radial_color", Color), ("radial_rotate", C.c_float), ("radial_invert", C.c_int),
        ("radial_bar_alias", C.c_float), ("radial_c_alias", C.c_float), ("radial_off_x", C.c_float), ("radial_off_y", C.c_float),
        ("circle_radius", C.c_float), ("circle_line", C.c_float), ("circle_outline", C.c_float * 4),
        ("circle_amplify", C.c_float), ("circle_rotate", C.c_float), ("circle_invert", C.c_int),
        ("circle_fill", C.c_int), ("circle_smooth", C.c_int),
        ("graph_vscale", C.c_float), ("graph_direction", C.c_int), ("graph_color", Color),
        ("graph_draw_outline", C.c_int), ("graph_draw_highlight", C.c_int), ("graph_outline", C.c_float * 4),
        ("graph_invert", C.c_int),
        ("wave_min_thickness", C.c_float), ("wave_max_thickness", C.c_float), ("wave_base_color", C.c_float * 4),
        ("wave_amplify", C.c_float), ("wave_outline", C.c_float * 4),
        ("rate_request", C.c_int), ("samplesize_request", C.c_int),
        ("fb_slots", C.c_int), ("lazy_smooth", C.c_int),
        ("bufscale", C.c_int), ("interpolate", C.c_int), ("fr", C.c_float), ("transform_smooth", C.c_int),
        ("smooth_distance", C.c_float), ("smooth_ratio", C.c_float),
        ("bars_color_prog", ColorProg), ("bars_outline_prog", ColorProg), ("radial_color_prog", ColorProg),
        ("graph_color_prog", ColorProg),
        ("clear_color", C.c_float * 4),
        ("radial_bar_width_int", C.c_int), ("radial_bar_outline_width", C.c_float), ("radial_bar_outline", C.c_float * 4),
        ("graph_join_channels", C.c_int), ("graph_anti_alias", C.c_int), ("shader_pre_smoothed", C.c_int),
        ("mirror_input", C.c_int),
    ]

    def copy(self):
        q = Params()
        C.memmove(C.byref(q), C.byref(self), C.sizeof(Params))
        return q

    @property
    def module_name(self):
        return MODULES[self.module]

    def to_dict(self):
        """JSON-serialisable copy (nested structs as dicts, arrays as lists); floats survive exactly"""
        def conv(v):
            if isinstance(v, ColorProg):                         # only the instructions in use
                return {"n_ops": v.n_ops, "result": v.result, "ops": [conv(v.ops[i]) for i in range(v.n_ops)]}
            if isinstance(v, C.Structure):
                return {n: conv(getattr(v, n)) for n, _t in v._fields_}
            if isinstance(v, C.Array):
                return [conv(x) for x in v]
            return v
        return conv(self)

    @classmethod
    def from_dict(cls, d):
        def fill(dst, src):
            for n, _t in dst._fields_:
                if n not in src:
                    continue
                cur = getattr(dst, n)
                if isinstance(cur, C.Structure):
                    fill(cur, src[n])
                elif isinstance(cur, C.Array):
                    for i, x in enumerate(src[n]):
                        if isinstance(cur[i], C.Structure):
                            fill(cur[i], x)
                        else:
                            cur[i] = x
                else:
                    setattr(dst, n, src[n])
        q = cls()
        fill(q, d)
        return q


class StreamStyle(C.Structure):
    """glava_b200_stream_style: what one stream overrides of the renderer's look (`set`: STYLE_* bits)"""
    _fields_ = [("set", C.c_uint32), ("amplify", C.c_float), ("fg", Color), ("bg", C.c_float * 4)]


STYLE_AMPLIFY, STYLE_FG, STYLE_BG = 1, 2, 4


class Export(C.Structure):
    """glava_b200_export: what one frame export writes — format (EXPORT_RGBA / _BGRA / _NV12), flags (EXPORT_OVER),
    the RGB8 background of the composite, and the destination's row pitch and NV12 CbCr plane offset (0: pitch * h)"""
    _fields_ = [("format", C.c_int), ("flags", C.c_uint32), ("background", C.c_uint8 * 4), ("pitch", C.c_size_t),
                ("uv_offset", C.c_size_t)]


class ExportScale(C.Structure):
    """glava_b200_export_scale: the source rectangle of a scaled export, top-down (all zero: the whole frame), and the
    output size"""
    _fields_ = [("src_x", C.c_int), ("src_y", C.c_int), ("src_w", C.c_int), ("src_h", C.c_int), ("out_w", C.c_int),
                ("out_h", C.c_int)]


class ExportRung(C.Structure):
    """glava_b200_export_rung: one rung of an encoder ladder — its destinations' descriptor and its scale rectangle"""
    _fields_ = [("desc", Export), ("scale", ExportScale)]


class Picture(C.Structure):
    """glava_b200_picture: one entry's plane pointers, each at the frame rectangle's first sample: Y; CbCr (NV12, P010) or
    Cb; Cr (the planar formats, else NULL)"""
    _fields_ = [("plane", C.c_void_p * 3)]


class OverlayPlanesDesc(C.Structure):
    """glava_b200_overlay_planes_desc: the picture format (EXPORT_NV12, _I420, _YUV444, _P010, _YUV420P10, _YUV444P10), the
    colour flags (EXPORT_FULL_RANGE / EXPORT_BT601), the luma pitch and the pitch of every chroma plane, in bytes"""
    _fields_ = [("format", C.c_int), ("flags", C.c_uint32), ("pitch", C.c_size_t), ("chroma_pitch", C.c_size_t)]


LADDER_MAX = 8
EXPORT_RGBA, EXPORT_BGRA, EXPORT_NV12 = 0, 1, 2
EXPORT_I420, EXPORT_YUV444, EXPORT_P010 = 4, 5, 6
EXPORT_YUV420P10, EXPORT_YUV444P10 = 7, 8                # planar 10-bit, LSB-aligned (yuv420p10le / yuv444p10le, DESIGN 4.16)
EXPORT_YUV422P, EXPORT_YUV422P10, EXPORT_UYVY = 10, 11, 12   # 4:2:2 (yuv422p / yuv422p10le / uyvy422, DESIGN 4.18)
EXPORT_YUVA420P, EXPORT_YUVA444P10 = 14, 15             # with an alpha plane (yuva420p / yuva444p10le, DESIGN 4.19)
EXPORT_OVER = 1
EXPORT_STRAIGHT = 4                                     # RGBA / BGRA with straight (unassociated) alpha (DESIGN 4.19)
EXPORT_FULL_RANGE, EXPORT_BT601 = 0x100, 0x200          # the Y'CbCr encoding (DESIGN 4.15); neither: BT.709 limited range
EXPORT_MATRICES = {"bt709": 0, "bt601": EXPORT_BT601}
EXPORT_PQ, EXPORT_HLG = 0x800, 0x1000                   # BT.2020 HDR, limited range, 10-bit formats only (DESIGN 4.22)
EXPORT_TRANSFERS = {"pq": EXPORT_PQ, "hlg": EXPORT_HLG}


def _colour_flags(matrix="bt709", full_range=False, transfer=None):
    """The colour flags of a Y'CbCr encoding: matrix "bt709" / "bt601" with full_range (DESIGN 4.15), or matrix "bt2020"
    with transfer "pq" / "hlg" (DESIGN 4.22: BT.2020 limited range HDR, P010 / YUV420P10 / YUV444P10 / YUV422P10; other
    formats reach the library's refusal).  Either of "bt2020" and transfer alone, and full_range with a transfer, raise
    ValueError"""
    if matrix == "bt2020" or transfer is not None:
        if matrix != "bt2020" or transfer not in EXPORT_TRANSFERS:
            raise ValueError(f"matrix {matrix!r}, transfer {transfer!r}: HDR is matrix='bt2020' with transfer 'pq' or 'hlg'")
        if full_range:
            raise ValueError(f"transfer {transfer!r}: HDR is limited range, full_range=True does not apply")
        return EXPORT_TRANSFERS[transfer]
    if matrix not in EXPORT_MATRICES:
        raise ValueError(f"matrix {matrix!r}: one of {sorted(EXPORT_MATRICES) + ['bt2020']}")
    return EXPORT_MATRICES[matrix] | (EXPORT_FULL_RANGE if full_range else 0)
EXPORT_FORMATS = {"rgba": EXPORT_RGBA, "bgra": EXPORT_BGRA, "nv12": EXPORT_NV12, "i420": EXPORT_I420,
                  "yuv444": EXPORT_YUV444, "p010": EXPORT_P010, "yuv420p10": EXPORT_YUV420P10,
                  "yuv444p10": EXPORT_YUV444P10, "yuv422p": EXPORT_YUV422P, "yuv422p10": EXPORT_YUV422P10,
                  "uyvy": EXPORT_UYVY, "yuva420p": EXPORT_YUVA420P, "yuva444p10": EXPORT_YUVA444P10}
OVERLAY_FORMATS = ("rgba", "bgra", "nv12")
# the formats overlay_planes takes: decoded pictures, one tensor per plane (DESIGN 4.17)
PLANES_FORMATS = ("nv12", "i420", "yuv444", "p010", "yuv420p10", "yuv444p10", "yuv422p", "yuv422p10", "uyvy")
# the formats whose samples are uint16, which also take uint16 `out` tensors
WIDE_FORMATS = ("p010", "yuv420p10", "yuv444p10", "yuv422p10", "yuva444p10")
# the formats with an alpha plane, returned as (Y, Cb, Cr, A)
ALPHA_FORMATS = ("yuva420p", "yuva444p10")


def _export_layout(fmt, w, h):
    """(rows, row bytes, pitch multiple) of one w x h output of `fmt` held as rows of one pitch: RGBA / BGRA h rows of w * 4
    bytes; NV12 / P010 h * 3 / 2 rows of w (P010: w uint16) samples, Y then CbCr; I420 / YUV420P10 h * 3 / 2 rows, the Y
    plane then the Cb and Cr planes back to back at pitch / 2 (pitch a multiple of 32); YUV444 / YUV444P10 3 h rows, the Y,
    Cb and Cr planes; YUV422P / YUV422P10 2 h rows, the Y plane then the Cb and Cr planes of h rows at pitch / 2 (pitch a
    multiple of 32); UYVY h rows of 2 w bytes; YUVA420P 5 h / 2 rows, I420's planes then the A plane of h rows at pitch
    (pitch a multiple of 32); YUVA444P10 4 h rows, the Y, Cb, Cr and A planes; the 10-bit formats hold w uint16 per row"""
    if fmt in ("rgba", "bgra"):
        return h, w * 4, 16
    if fmt == "uyvy":
        return h, w * 2, 16
    row = w * 2 if fmt in WIDE_FORMATS else w
    if fmt == "yuva420p":
        return h * 5 // 2, row, 32
    if fmt == "yuva444p10":
        return 4 * h, row, 16
    if fmt in ("yuv444", "yuv444p10"):
        return 3 * h, row, 16
    if fmt in ("yuv422p", "yuv422p10"):
        return 2 * h, row, 32
    return h * 3 // 2, row, 32 if fmt in ("i420", "yuv420p10") else 16


def _export_views(fmt, t, w, h):
    """what an export into t returns: t is uint8 [..., rows, pitch] with contiguous rows as _export_layout describes.  RGBA /
    BGRA [..., h, w, 4], NV12 [..., h * 3 / 2, w] uint8, P010 [..., h * 3 / 2, w] uint16, I420 / YUV444 the plane views
    (Y, Cb, Cr), each [..., rows, cols], YUV420P10 / YUV444P10 the same as uint16; YUV422P / YUV422P10 (Y, Cb, Cr) with
    Cb and Cr [..., h, w / 2]; UYVY [..., h, 2 w] uint8 (Cb, Y0, Cr, Y1 per pixel pair); YUVA420P / YUVA444P10 (Y, Cb, Cr,
    A) as I420 / YUV444P10 with A [..., h, w] (uint8 / uint16) after Cr"""
    import torch
    if fmt in ("rgba", "bgra"):
        return t[..., :w * 4].unflatten(-1, (w, 4))
    if fmt == "uyvy":
        return t[..., :w * 2]
    if fmt == "nv12":
        return t[..., :w]
    if fmt in WIDE_FORMATS:
        t = t.view(torch.uint16)
    if fmt == "p010":
        return t[..., :w]
    P = t.shape[-1]                                           # the pitch in samples
    flat = t.flatten(-2)
    cw, ch, cp = ((w // 2, h // 2, P // 2) if fmt in ("i420", "yuv420p10", "yuva420p") else (w // 2, h, P // 2)
                  if fmt in ("yuv422p", "yuv422p10") else (w, h, P))
    n = ch * cp
    y = flat[..., :P * h].unflatten(-1, (h, P))[..., :w]
    cb = flat[..., P * h:P * h + n].unflatten(-1, (ch, cp))[..., :cw]
    cr = flat[..., P * h + n:P * h + 2 * n].unflatten(-1, (ch, cp))[..., :cw]
    if fmt in ALPHA_FORMATS:
        return y, cb, cr, flat[..., P * h + 2 * n:2 * P * h + 2 * n].unflatten(-1, (h, P))[..., :w]
    return y, cb, cr


_lib = None


def lib_path():
    return os.path.join(_HERE, "libglava_b200.so")


def lib():
    """Load libglava_b200.so (built in-tree by __graft_entry__.build()).  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise GlavaError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(the GPU path has no CPU fallback)")
    L = C.CDLL(path)
    vp, cp, i32 = C.c_void_p, C.c_char_p, C.c_int
    L.glava_b200_last_error.restype = cp
    L.glava_b200_version.restype = cp
    L.glava_b200_default_params.argtypes = [C.POINTER(Params), cp]
    L.glava_b200_load_config.argtypes = [C.POINTER(Params), C.POINTER(cp), cp, C.POINTER(cp), cp]
    L.glava_b200_load_config_binds.argtypes = [C.POINTER(Params), C.POINTER(cp), cp, C.POINTER(cp), cp, C.POINTER(cp)]
    L.glava_b200_reconfigure.argtypes = [vp, C.POINTER(Params)]
    L.glava_b200_new.restype = vp
    L.glava_b200_new.argtypes = [C.POINTER(Params), i32, i32]
    L.glava_b200_destroy.argtypes = [vp]
    L.glava_b200_get_params.argtypes = [vp, C.POINTER(Params)]
    L.glava_b200_batch.argtypes = [vp]
    L.glava_b200_module_name.argtypes = [vp]
    L.glava_b200_module_name.restype = cp
    L.glava_b200_host_alloc.restype = vp
    L.glava_b200_host_alloc.argtypes = [C.c_size_t]
    L.glava_b200_host_free.argtypes = [vp]
    L.glava_b200_host_alloc_on.restype = vp
    L.glava_b200_host_alloc_on.argtypes = [C.c_size_t, i32]
    L.glava_b200_device_numa_node.argtypes = [i32]
    L.glava_b200_bind_thread_to_device.argtypes = [i32]
    L.glava_b200_shard_range.argtypes = [i32, i32, i32, C.POINTER(i32), C.POINTER(i32)]
    L.glava_b200_new_sharded.restype = vp
    L.glava_b200_new_sharded.argtypes = [C.POINTER(Params), i32, C.c_uint64]
    L.glava_b200_new_sharded_devices.restype = vp
    L.glava_b200_new_sharded_devices.argtypes = [C.POINTER(Params), i32, C.POINTER(i32), i32]
    L.glava_b200_sharded_destroy.argtypes = [vp]
    L.glava_b200_sharded_shards.argtypes = [vp]
    L.glava_b200_sharded_batch.argtypes = [vp]
    L.glava_b200_sharded_shard.restype = vp
    L.glava_b200_sharded_shard.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.glava_b200_sharded_update.argtypes = [vp, vp, vp, C.c_size_t, vp]
    L.glava_b200_sharded_rerender.argtypes = [vp]
    L.glava_b200_sharded_ingest_fifo.argtypes = [vp, vp, i32]
    L.glava_b200_sharded_sync.argtypes = [vp]
    L.glava_b200_sharded_readback.argtypes = [vp, i32, vp]
    L.glava_b200_sharded_frame_device.restype = vp
    L.glava_b200_sharded_frame_device.argtypes = [vp, i32, C.POINTER(i32)]
    L.glava_b200_sharded_textures.argtypes = [vp, vp, vp]
    L.glava_b200_set_async_input.argtypes = [vp, i32]
    L.glava_b200_wait_input.argtypes = [vp]
    L.glava_b200_update.argtypes = [vp, vp, vp, C.c_size_t, i32]
    L.glava_b200_update_device.argtypes = [vp, vp, vp, C.c_size_t, i32]
    L.glava_b200_update_device_after.argtypes = [vp, vp, vp, C.c_size_t, i32, vp]
    L.glava_b200_input_event.restype = vp
    L.glava_b200_input_event.argtypes = [vp]
    L.glava_b200_update_masked.argtypes = [vp, vp, vp, C.c_size_t, vp]
    L.glava_b200_update_device_masked.argtypes = [vp, vp, vp, C.c_size_t, vp]
    L.glava_b200_update_rings_masked.argtypes = [vp, vp]
    L.glava_b200_ingest_fifo.argtypes = [vp, vp, i32]
    L.glava_b200_ingest_float.argtypes = [vp, vp, i32]
    L.glava_b200_update_rings.argtypes = [vp, i32]
    L.glava_b200_sync.argtypes = [vp]
    L.glava_b200_readback.argtypes = [vp, i32, vp]
    L.glava_b200_readback_async.argtypes = [vp, i32, vp]
    L.glava_b200_readback_fence.argtypes = [vp]
    L.glava_b200_spectrum.argtypes = [vp, vp, vp]
    L.glava_b200_textures.argtypes = [vp, vp, vp]
    L.glava_b200_framebuffer_device.argtypes = [vp]
    L.glava_b200_framebuffer_device.restype = vp
    L.glava_b200_cuda_stream.argtypes = [vp]
    L.glava_b200_cuda_stream.restype = vp
    L.glava_b200_smooth_pass.argtypes = [vp, vp, vp, i32]
    L.glava_b200_raster_textures.argtypes = [vp, vp, vp]
    L.glava_b200_transform_smooth.argtypes = [vp, vp, i32]
    L.glava_b200_timeline.argtypes = [vp, vp, i32, C.POINTER(i32), C.POINTER(i32)]
    L.glava_b200_sizereq.argtypes = [vp, i32, i32]
    L.glava_b200_wait_frame.argtypes = [vp]
    L.glava_b200_frame_event.argtypes = [vp]
    L.glava_b200_frame_event.restype = vp
    L.glava_b200_frame_device.argtypes = [vp, i32]
    L.glava_b200_frame_device.restype = vp
    L.glava_b200_framebuffer_ipc.argtypes = [vp, vp, C.c_size_t]
    L.glava_b200_spectrum_size.argtypes = [vp]
    L.glava_b200_launch_count.argtypes = [vp]
    L.glava_b200_launch_count.restype = C.c_uint64
    L.glava_b200_set_abort_hook.argtypes = [vp]
    L.glava_b200_set_timing.argtypes = [vp, i32]
    L.glava_b200_kernel_times.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i32), C.POINTER(C.c_double), C.POINTER(i32)]
    L.glava_b200_pipe_new.restype = vp
    L.glava_b200_pipe_new.argtypes = [C.POINTER(cp), cp, C.POINTER(cp), cp, C.POINTER(cp)]
    L.glava_b200_pipe_feed.argtypes = [vp, cp, C.c_size_t]
    L.glava_b200_pipe_params.argtypes = [vp, C.POINTER(Params)]
    L.glava_b200_pipe_bind_count.argtypes = [vp]
    L.glava_b200_pipe_bind.argtypes = [vp, i32, C.POINTER(cp), C.POINTER(cp), C.POINTER(C.c_float)]
    L.glava_b200_pipe_apply.argtypes = [vp, vp]
    L.glava_b200_pipe_free.argtypes = [vp]
    L.glava_b200_stream_state_bytes.restype = C.c_size_t
    L.glava_b200_stream_state_bytes.argtypes = [C.POINTER(Params)]
    L.glava_b200_reset_streams.argtypes = [vp, vp]
    L.glava_b200_save_streams.argtypes = [vp, vp, i32, vp]
    L.glava_b200_load_streams.argtypes = [vp, vp, i32, vp]
    L.glava_b200_sharded_reset_streams.argtypes = [vp, vp]
    L.glava_b200_sharded_save_streams.argtypes = [vp, vp, i32, vp]
    L.glava_b200_sharded_load_streams.argtypes = [vp, vp, i32, vp]
    L.glava_b200_style_params.argtypes = [C.POINTER(Params), C.POINTER(StreamStyle), C.POINTER(Params)]
    L.glava_b200_parse_hex_color.argtypes = [C.c_char_p, C.POINTER(C.c_float)]
    for f in ("glava_b200_set_stream_styles", "glava_b200_get_stream_styles", "glava_b200_sharded_set_stream_styles",
              "glava_b200_sharded_get_stream_styles"):
        getattr(L, f).argtypes = [vp, vp, i32, vp]
    L.glava_b200_export_bytes.argtypes = [vp, C.POINTER(Export), C.POINTER(C.c_size_t)]
    L.glava_b200_export_frames.argtypes = [vp, vp, i32, vp, C.POINTER(Export), vp, vp]
    L.glava_b200_sharded_export_frames.argtypes = [vp, vp, i32, vp, C.POINTER(Export)]
    L.glava_b200_export_scaled_bytes.argtypes = [vp, C.POINTER(Export), C.POINTER(ExportScale), C.POINTER(C.c_size_t)]
    L.glava_b200_export_scaled.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export), C.POINTER(ExportScale), vp, vp]
    L.glava_b200_sharded_export_scaled.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export), C.POINTER(ExportScale)]
    L.glava_b200_overlay_frames.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export), vp, vp]
    L.glava_b200_sharded_overlay_frames.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export)]
    L.glava_b200_export_ladder.argtypes = [vp, vp, i32, C.POINTER(ExportRung), i32, vp, vp, vp, vp]
    L.glava_b200_sharded_export_ladder.argtypes = [vp, vp, i32, C.POINTER(ExportRung), i32, vp, vp]
    L.glava_b200_overlay_planes.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), vp, vp]
    L.glava_b200_sharded_overlay_planes.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc)]
    L.glava_b200_overlay_frames_opacity.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export), vp, vp, vp]
    L.glava_b200_sharded_overlay_frames_opacity.argtypes = [vp, vp, i32, vp, vp, C.POINTER(Export), vp]
    L.glava_b200_overlay_planes_opacity.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), vp, vp, vp]
    L.glava_b200_sharded_overlay_planes_opacity.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), vp]
    L.glava_b200_overlay_scaled.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc), C.POINTER(ExportScale),
                                            vp, vp, vp]
    L.glava_b200_sharded_overlay_scaled.argtypes = [vp, vp, i32, C.POINTER(Picture), C.POINTER(OverlayPlanesDesc),
                                                    C.POINTER(ExportScale), vp]
    _lib = L
    # errors surface as Python exceptions; keep stderr quiet
    _quiet = C.CFUNCTYPE(None, cp)(lambda msg: None)
    L._quiet_hook = _quiet
    L.glava_b200_set_abort_hook(C.cast(_quiet, vp))
    return L


def _check(rc):
    if rc != 0:
        raise GlavaError(lib().glava_b200_last_error().decode(errors="replace") or f"error {rc}")


def default_params(module="bars", **overrides):
    p = Params()
    _check(lib().glava_b200_default_params(C.byref(p), module.encode()))
    for k, v in overrides.items():
        if isinstance(v, (list, tuple)):
            v = type(getattr(p, k))(*v)
        setattr(p, k, v)
    return p


STATE_HEADER_BYTES = 4096        # GLAVA_B200_STATE_HEADER_BYTES


def stream_state_bytes(params):
    """bytes of one stream's state blob for renderers created with `params` (glava_b200_stream_state_bytes); raises while
    keyframe interpolation is active"""
    n = lib().glava_b200_stream_state_bytes(C.byref(params))
    if n == 0:
        raise GlavaError(lib().glava_b200_last_error().decode(errors="replace"))
    return int(n)


class _StreamState:
    """reset_streams / save_streams / load_streams over the handle's C entry points (self._fn: their names)"""

    def _stream_list(self, streams):
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        assert s.ndim == 1
        return s

    def reset_streams(self, mask):
        """streams with mask[s] != 0 start fresh: from their next update on, what a new batch-1 renderer renders"""
        m = np.ascontiguousarray(np.asarray(mask) != 0, dtype=np.uint8)
        assert m.shape == (self.batch,), m.shape
        _check(self._fn[0](self._h, m.ctypes.data))

    def save_streams(self, streams):
        """-> uint8 [len(streams)][stream_state_bytes] blobs of the listed streams' state"""
        s = self._stream_list(streams)
        out = np.empty((s.shape[0], stream_state_bytes(self.params)), np.uint8)
        _check(self._fn[1](self._h, s.ctypes.data, s.shape[0], out.ctypes.data))
        return out

    def load_streams(self, streams, blobs):
        """put blobs from save_streams (same effective parameters, any renderer) into the listed streams"""
        s = self._stream_list(streams)
        b = np.ascontiguousarray(blobs, dtype=np.uint8)
        assert b.shape == (s.shape[0], stream_state_bytes(self.params)), b.shape
        _check(self._fn[2](self._h, s.ctypes.data, s.shape[0], b.ctypes.data))


def _cstr_array(items):
    if items is None:
        return None
    arr = (C.c_char_p * (len(items) + 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode()
    arr[len(items)] = None
    return arr


def load_config(paths=None, entry="rc.glsl", requests=None, force_module=None, binds=None):
    """rd_new's config half (render.c:1322-1435): read `entry` from the first of `paths`, apply
    `#request`s and `requests` (CLI --request strings), then the module's `#define`s.
    binds: {"fg": "#ff0000", ...} — `--pipe` binds resolving `@name:default` macros."""
    p = Params()
    bl = [f"{k}={v}" for k, v in binds.items()] if binds else None
    _check(lib().glava_b200_load_config_binds(C.byref(p), _cstr_array(paths), entry.encode() if entry else None,
                                              _cstr_array(requests), force_module.encode() if force_module else None,
                                              _cstr_array(bl)))
    return p


def _rgba(value):
    """a colour as floats: "#rrggbb[aa]" through the library's own parser (glava_b200_parse_hex_color: the rounding of a
    `--pipe` bind), or 4 numbers"""
    if isinstance(value, str):
        out = (C.c_float * 4)()
        _check(lib().glava_b200_parse_hex_color(value.strip().encode(), out))
        return tuple(out)
    v = tuple(float(x) for x in value)
    assert len(v) == 4, value
    return v


def stream_style(style):
    """a StreamStyle from a StreamStyle, None (no style) or a dict such as
    {"amplify": 450, "fg": "#ff8000", "bg": (0.1, 0.1, 0.1, 1)}; fg may also be a Color (mode 0: a gradient)"""
    if isinstance(style, StreamStyle):
        return style
    s = StreamStyle()
    if not style:
        return s
    unknown = set(style) - {"amplify", "fg", "bg"}
    if unknown:
        raise ValueError(f"unknown stream style fields {sorted(unknown)}")
    if style.get("amplify") is not None:
        s.set |= STYLE_AMPLIFY
        s.amplify = float(style["amplify"])
    if style.get("fg") is not None:
        s.set |= STYLE_FG
        fg = style["fg"]
        if isinstance(fg, Color):
            C.memmove(C.byref(s.fg), C.byref(fg), C.sizeof(Color))
        else:
            c = _rgba(fg)
            s.fg.mode = 1
            s.fg.lo = (C.c_float * 4)(*c)
            s.fg.hi = (C.c_float * 4)(*c)
    if style.get("bg") is not None:
        s.set |= STYLE_BG
        s.bg = (C.c_float * 4)(*_rgba(style["bg"]))
    return s


def style_params(params, style):
    """`params` with the stream style applied (glava_b200_style_params): what a batch-1 renderer needs to render what a
    stream of that style renders"""
    out = Params()
    s = stream_style(style)
    _check(lib().glava_b200_style_params(C.byref(params), C.byref(s), C.byref(out)))
    return out


class _StreamStyles:
    """set_stream_styles / get_stream_styles over the handle's C entry points (self._style_fn: set, get)"""

    def set_stream_styles(self, streams, styles):
        """give streams[i] the look styles[i] (StreamStyle, dict or None = the renderer's own) from the next raster pass on"""
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        styles = list(styles)
        assert len(styles) == s.shape[0], (len(styles), s.shape)
        arr = (StreamStyle * max(len(styles), 1))(*[stream_style(x) for x in styles])
        _check(self._style_fn[0](self._h, s.ctypes.data, s.shape[0], arr))

    def get_stream_styles(self, streams):
        """-> [StreamStyle] of the listed streams (set == 0: none)"""
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        arr = (StreamStyle * max(s.shape[0], 1))()
        _check(self._style_fn[1](self._h, s.ctypes.data, s.shape[0], arr))
        return [arr[i] for i in range(s.shape[0])]


class _FrameExport:
    """export_frames over the handle's C entry point: destinations as torch tensors (DESIGN 4.10)"""

    def _export_plan(self, streams, fmt, over, background, out, device_of, size=None, matrix="bt709", full_range=False,
                     straight=False, transfer=None):
        """-> (stream list, Export, [dst pointers], what to return).  device_of(stream): the CUDA device of a stream's
        frame.  size: (w, h) of each output, None: the frame's.  out: None (allocate), one uint8 tensor [count, rows, ...]
        whose dim 1 steps by the pitch, or a list of count tensors [rows, ...] with one common pitch; rows as
        _export_layout gives them (h for RGBA / BGRA and UYVY, h * 3 / 2 for NV12, I420, P010 and YUV420P10, 2 h for YUV422P
        and YUV422P10, 3 h for YUV444 and YUV444P10; the planar formats keep their planes back to back from row h); P010,
        YUV420P10, YUV444P10 and YUV422P10 also take uint16 tensors.  matrix / full_range: the Y'CbCr encoding, straight:
        straight alpha (_export_desc)"""
        import torch
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        count = int(s.shape[0])
        devices = [device_of(int(x)) for x in s]
        p = self.params
        w, h = (p.w, p.h) if size is None else (int(size[0]), int(size[1]))
        desc = _export_desc(fmt, over, background, matrix, full_range, straight, transfer)
        rows, row_bytes, align = _export_layout(fmt, w, h)
        dtypes = (torch.uint8, torch.uint16) if fmt in WIDE_FORMATS else (torch.uint8,)

        if out is None:
            pitch = (row_bytes + align - 1) // align * align
            if len(set(devices)) <= 1:
                base = torch.empty((count, rows, pitch), dtype=torch.uint8, device=f"cuda:{devices[0] if devices else 0}")
                dst = [base.data_ptr() + i * rows * pitch for i in range(count)]
                result = _export_views(fmt, base, w, h)
            else:
                bufs = [torch.empty((rows, pitch), dtype=torch.uint8, device=f"cuda:{d}") for d in devices]
                dst = [b.data_ptr() for b in bufs]
                result = [_export_views(fmt, b, w, h) for b in bufs]
        else:
            tensors = list(out) if isinstance(out, (list, tuple)) else None
            if tensors is None:
                if out.dtype not in dtypes or not out.is_cuda or out.dim() < 3 or out.shape[0] != count or out.shape[1] != rows:
                    raise ValueError(f"out: a uint8 CUDA tensor [{count}, {rows}, ...] (got {out.dtype} {tuple(out.shape)})")
                pitch = out.stride(1) * out.element_size()
                dst = [out.data_ptr() + i * out.stride(0) * out.element_size() for i in range(count)]
                row = out[0, 0]
            else:
                if len(tensors) != count:
                    raise ValueError(f"out: {count} tensors, got {len(tensors)}")
                for t in tensors:
                    if (t.dtype != tensors[0].dtype or t.dtype not in dtypes or not t.is_cuda or t.dim() < 2 or t.shape[0] != rows
                            or t.stride(0) != tensors[0].stride(0)):
                        raise ValueError(f"out: uint8 CUDA tensors [{rows}, ...] with one pitch (got {t.dtype} {tuple(t.shape)})")
                pitch = tensors[0].stride(0) * tensors[0].element_size()
                dst = [t.data_ptr() for t in tensors]
                row = tensors[0][0]
            if not row.is_contiguous() or row.numel() * row.element_size() < row_bytes:
                raise ValueError(f"out: every row must hold {row_bytes} contiguous bytes")
            result = out
        desc.pitch = pitch
        desc.uv_offset = pitch * h if fmt in ("nv12", "p010") else 0
        return s, desc, (C.c_void_p * max(count, 1))(*dst), result

    def _ladder_plan(self, streams, rungs, out, device_of):
        """-> (stream list, ExportRung array, nrungs, [count][nrungs] dst pointers, [one result per rung]) of an encoder
        ladder (DESIGN 4.13): each rung planned by _export_plan as export_scaled plans it.  rungs: dicts with export_scaled's
        keywords size (None: the frame's), crop, fmt (default "nv12"), over, background, matrix and full_range; out: None
        or one entry per rung in any form export_scaled takes"""
        rungs = list(rungs)
        outs = [None] * len(rungs) if out is None else list(out)
        if len(outs) != len(rungs):
            raise ValueError(f"out: one entry per rung ({len(rungs)}), got {len(outs)}")
        p = self.params
        s = np.ascontiguousarray(np.asarray(list(streams), dtype=np.int64).reshape(-1), dtype=np.int32)
        arr = (ExportRung * max(len(rungs), 1))()
        ptrs, results = [], []
        for j, (rung, o) in enumerate(zip(rungs, outs)):
            unknown = set(rung) - {"size", "crop", "fmt", "over", "background", "matrix", "full_range", "straight",
                                   "transfer"}
            if unknown:
                raise ValueError(f"rungs[{j}]: unknown keys {sorted(unknown)}")
            size = rung.get("size") or (p.w, p.h)
            _, desc, dst, result = self._export_plan(s, rung.get("fmt", "nv12"), rung.get("over", False),
                                                     rung.get("background", (0, 0, 0)), o, device_of, size,
                                                     rung.get("matrix", "bt709"), rung.get("full_range", False),
                                                     rung.get("straight", False), rung.get("transfer"))
            arr[j].desc, arr[j].scale = desc, _export_scale(size, rung.get("crop"))
            ptrs.append(dst)
            results.append(result)
        count, n = int(s.shape[0]), len(rungs)
        dst = (C.c_void_p * max(count * n, 1))(*[ptrs[j][i] for i in range(count) for j in range(n)])
        return s, arr, n, dst, results

    @staticmethod
    def _opacity(opacity, count):
        """-> None (opacity None) or the uint8 [count] opacities K = floor(255 o + 0.5) of an overlay (DESIGN 4.20).  opacity:
        one float for every entry, or a sequence / 1-D array of `count` floats, each in [0, 1].  Raises ValueError for NaN,
        a value outside [0, 1] or a wrong length."""
        if opacity is None:
            return None
        if hasattr(opacity, "detach"):                        # a torch tensor, possibly on the device
            opacity = opacity.detach().cpu().numpy()
        o = np.asarray(opacity, dtype=np.float64)
        if o.ndim == 0:
            o = np.full(count, float(o))
        elif o.ndim != 1 or o.shape[0] != count:
            raise ValueError(f"opacity: one float or {count} of them, got shape {o.shape}")
        if np.isnan(o).any():
            raise ValueError("opacity: NaN")
        if (o < 0).any() or (o > 1).any():
            raise ValueError(f"opacity: values must lie in [0, 1] (got {o.min()} .. {o.max()})")
        return np.ascontiguousarray(np.floor(255.0 * o + 0.5), dtype=np.uint8)

    @staticmethod
    def _overlay_scale(size, crop):
        """-> (None, None) when size and crop are None (the overlay at the frame's own size), else (rectangle size (w, h),
        ExportScale) of an overlay of the downscaled, cropped frame (DESIGN 4.21): size = (w, h), None: the crop's size; crop
        = (x, y, w, h) in top-down coordinates, None: the whole frame.  Raises ValueError for a size that is not two
        positive integers or a crop that is not four integers (the library refuses a crop that leaves the frame and
        upscaling)."""
        if size is None and crop is None:
            return None, None
        if crop is not None:
            crop = tuple(int(v) for v in crop)
            if len(crop) != 4:
                raise ValueError(f"crop: (x, y, w, h), got {crop}")
        size = crop[2:] if size is None else tuple(int(v) for v in size)
        if len(size) != 2 or min(size) < 1:
            raise ValueError(f"size: (w, h) of positive integers, got {size}")
        return size, _export_scale(size, crop)

    @staticmethod
    def _frames_pictures(desc, dst, uv, count):
        """overlay_frames' (Export, dst, dst_uv) as glava_b200_overlay_scaled's (OverlayPlanesDesc, Picture array): RGBA /
        BGRA one plane, NV12 its Y and CbCr planes at one pitch"""
        pd = OverlayPlanesDesc()
        pd.format, pd.flags, pd.pitch = desc.format, desc.flags, desc.pitch
        pd.chroma_pitch = desc.pitch if uv is not None else 0
        arr = (Picture * max(count, 1))()
        for i in range(count):
            arr[i].plane = (C.c_void_p * 3)(dst[i], uv[i] if uv is not None else None, None)
        return pd, arr

    def _overlay_plan(self, streams, images, at, fmt, matrix="bt709", full_range=False, size=None):
        """-> (stream list, Export, dst pointers, dst_uv pointers or None) of an overlay (DESIGN 4.12).  images: one uint8
        CUDA tensor per entry (one may repeat) or one [count, ...] tensor, each [H, W, 4] (RGBA / BGRA) or [H * 3 / 2, W]
        (NV12, CbCr rows from row H) with contiguous rows and one pitch for all; at: (x, y) of each frame's top-left
        corner in its image (None: (0, 0)).  Raises ValueError for a rectangle that leaves its image or whose rows do
        not start at multiples of 16 bytes (the device refuses the rest).  matrix / full_range: the encoding of an NV12
        picture (_export_desc).  size: the rectangle's (w, h), None: the frame's."""
        import torch
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        count = int(s.shape[0])
        if fmt not in OVERLAY_FORMATS:
            raise ValueError(f"format {fmt!r}: the overlay takes one of {list(OVERLAY_FORMATS)}")
        nv12 = fmt == "nv12"

        def describe(t, what):
            """-> (H, W, pitch) of one image"""
            if t.dtype != torch.uint8 or not t.is_cuda or t.dim() != (2 if nv12 else 3) or (not nv12 and t.shape[2] != 4):
                raise ValueError(f"{what}: a uint8 CUDA tensor {'[H * 3 / 2, W]' if nv12 else '[H, W, 4]'} "
                                 f"(got {t.dtype} {tuple(t.shape)})")
            if (nv12 and t.stride(1) != 1) or (not nv12 and (t.stride(1), t.stride(2)) != (4, 1)):
                raise ValueError(f"{what}: rows must be contiguous")
            H, W = (t.shape[0] * 2 // 3, t.shape[1]) if nv12 else (t.shape[0], t.shape[1])
            if nv12 and (t.shape[0] % 3 or H % 2):
                raise ValueError(f"{what}: NV12 has H * 3 / 2 rows with H even (got {t.shape[0]})")
            return H, W, t.stride(0)

        # per entry: (base address, H, W, pitch), each image described once (1024 entries cost no 1024 tensor views)
        if isinstance(images, (list, tuple)):
            seen, ents = {}, []
            for i, t in enumerate(images):
                if id(t) not in seen:
                    seen[id(t)] = (t.data_ptr(),) + describe(t, f"images[{i}]")
                ents.append(seen[id(t)])
        else:
            if images.dim() < 1 or images.shape[0] != count:
                raise ValueError(f"images: {count} images, got a tensor {tuple(images.shape)}")
            one = describe(images[0], "images[0]") if count else None
            ents = [(images.data_ptr() + i * images.stride(0),) + one for i in range(count)]
        if len(ents) != count:
            raise ValueError(f"images: {count} images, got {len(ents)}")
        at = [(0, 0)] * count if at is None else [(int(x), int(y)) for x, y in at]
        if len(at) != count:
            raise ValueError(f"at: {count} positions, got {len(at)}")
        w, h = size or (self.params.w, self.params.h)
        px = 1 if nv12 else 4
        dst, uv, pitch = [], [], None
        for i, ((base, H, W, ip), (x, y)) in enumerate(zip(ents, at)):
            if pitch is None:
                pitch = ip
            elif ip != pitch:
                raise ValueError(f"images[{i}]: pitch {ip}, the others {pitch}: one pitch per call")
            if x < 0 or y < 0 or x + w > W or y + h > H:
                raise ValueError(f"images[{i}]: the {w}x{h} frame at ({x}, {y}) leaves the {W}x{H} image")
            d = base + y * pitch + x * px
            u = base + (H + y // 2) * pitch + x if nv12 else None
            if d % 16 or (nv12 and (y % 2 or u % 16)):
                raise ValueError(f"images[{i}]: the frame at ({x}, {y}) does not start at a multiple of 16 bytes"
                                 + (" on an even row" if nv12 else ""))
            dst.append(d)
            uv.append(u)
        desc = _export_desc(fmt, False, (0, 0, 0), matrix, full_range)
        desc.pitch = pitch or 0
        arr = (C.c_void_p * max(count, 1))(*dst)
        return s, desc, arr, (C.c_void_p * max(count, 1))(*uv) if nv12 else None

    def _planes_plan(self, streams, pictures, at, fmt, matrix="bt709", full_range=False, size=None, transfer=None):
        """-> (stream list, OverlayPlanesDesc, Picture array) of an overlay onto decoded pictures (DESIGN 4.17).  pictures:
        one tuple of plane tensors per entry (a tuple may repeat), or one tuple of batched [count, rows, cols] plane tensors;
        a tuple is (Y, CbCr) for NV12 and P010, (Y, Cb, Cr) otherwise, each CUDA, uint8 (the 8-bit formats) or uint16 or
        uint8 with doubled width (the 10-bit formats), with contiguous rows: Y [H, W], NV12 CbCr [H / 2, W] bytes, P010 CbCr
        [H / 2, W] samples, I420 / YUV420P10 Cb and Cr [H / 2, W / 2], YUV444 / YUV444P10 Cb and Cr [H, W], YUV422P /
        YUV422P10 Cb and Cr [H, W / 2] (export_frames' plane views); UYVY is one plane [H, 2 W] of bytes, given as a tensor
        or a 1-tuple (one [count, H, 2 W] tensor for a batch), and a 4:2:2 frame starts at an even x.  Every luma plane has one pitch and every chroma plane one pitch.  at: (x, y) of each frame's top-left
        in luma samples (None: (0, 0)).  Raises ValueError for a rectangle that leaves its picture, mixed pitches within a
        plane kind, or a plane start that is not 16-byte aligned (the library refuses the rest).  size: the rectangle's (w, h),
        None: the frame's."""
        import torch
        if fmt not in PLANES_FORMATS:
            raise ValueError(f"format {fmt!r}: overlay_planes takes one of {list(PLANES_FORMATS)} "
                             "(RGBA and BGRA images go to overlay_frames)")
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        count = int(s.shape[0])
        nplanes = 2 if fmt in ("nv12", "p010") else 1 if fmt == "uyvy" else 3
        sb = 2 if fmt in WIDE_FORMATS else 1                  # bytes per sample
        px = 2 if fmt == "uyvy" else sb                       # luma-plane bytes per pixel (UYVY: its one packed plane)
        c420 = fmt in ("nv12", "i420", "p010", "yuv420p10")
        c422 = fmt in ("yuv422p", "yuv422p10", "uyvy")

        def describe(planes, what, batched):
            """-> ([base address per plane], H, W, pitch, chroma pitch) of one picture (batched: of entry 0)"""
            planes = (planes,) if isinstance(planes, torch.Tensor) else tuple(planes)
            if len(planes) != nplanes:
                raise ValueError(f"{what}: {fmt} has {nplanes} planes, got {len(planes)}")
            dims = 3 if batched else 2
            bases, shapes, pitches = [], [], []
            for p, t in enumerate(planes):
                ok = t.dtype in ((torch.uint8, torch.uint16) if sb == 2 else (torch.uint8,))
                if not ok or not t.is_cuda or t.dim() != dims:
                    raise ValueError(f"{what}[{p}]: a {'uint16 or uint8' if sb == 2 else 'uint8'} CUDA tensor of {dims} "
                                     f"dimensions (got {t.dtype} {tuple(t.shape)})")
                if t.stride(-1) != 1:
                    raise ValueError(f"{what}[{p}]: rows must be contiguous")
                if batched and t.shape[0] != count:
                    raise ValueError(f"{what}[{p}]: {count} pictures, got {t.shape[0]}")
                bases.append(t.data_ptr())
                shapes.append((t.shape[-2], t.shape[-1] * t.element_size()))   # rows, row bytes
                pitches.append(t.stride(-2) * t.element_size())
            H, W = shapes[0][0], shapes[0][1] // px
            crows = H // 2 if c420 else H
            cbytes = {"nv12": W, "p010": 2 * W, "i420": W // 2, "yuv420p10": W, "yuv444": W, "yuv444p10": 2 * W,
                      "yuv422p": W // 2, "yuv422p10": W, "uyvy": 0}[fmt]
            for p in range(1, nplanes):
                if shapes[p][0] != crows or shapes[p][1] < cbytes:
                    raise ValueError(f"{what}[{p}]: a {W}x{H} {fmt} picture has chroma planes of {crows} rows of {cbytes} "
                                     f"bytes (got {shapes[p][0]} rows of {shapes[p][1]})")
            if nplanes == 3 and pitches[1] != pitches[2]:
                raise ValueError(f"{what}: Cb pitch {pitches[1]}, Cr pitch {pitches[2]}: one chroma pitch per call")
            steps = [t.stride(0) * t.element_size() for t in planes] if batched else None
            return bases, H, W, pitches[0], pitches[1] if nplanes > 1 else 0, steps

        if fmt == "uyvy" and isinstance(pictures, torch.Tensor):  # UYVY: one batched tensor
            pictures = (pictures,)
        if fmt == "uyvy" and isinstance(pictures, (list, tuple)) and len(pictures) and isinstance(pictures[0], torch.Tensor) \
                and pictures[0].dim() == 2:                   # one [H, 2W] tensor per picture
            pictures = [(t,) for t in pictures]
        if isinstance(pictures, (list, tuple)) and len(pictures) and isinstance(pictures[0], torch.Tensor):
            bases, H, W, P, CP, steps = describe(pictures, "pictures", True)
            ents = [([b + i * st for b, st in zip(bases, steps)], H, W, P, CP) for i in range(count)]
        else:
            seen, ents = {}, []
            for i, pic in enumerate(pictures):
                if id(pic) not in seen:
                    seen[id(pic)] = describe(pic, f"pictures[{i}]", False)[:5]
                ents.append(seen[id(pic)])
        if len(ents) != count:
            raise ValueError(f"pictures: {count} pictures, got {len(ents)}")
        at = [(0, 0)] * count if at is None else [(int(x), int(y)) for x, y in at]
        if len(at) != count:
            raise ValueError(f"at: {count} positions, got {len(at)}")
        w, h = size or (self.params.w, self.params.h)
        arr = (Picture * max(count, 1))()
        pitch = cpitch = None
        for i, ((bases, H, W, P, CP), (x, y)) in enumerate(zip(ents, at)):
            if pitch is None:
                pitch, cpitch = P, CP
            elif (P, CP) != (pitch, cpitch):
                raise ValueError(f"pictures[{i}]: pitches {P} / {CP}, the others {pitch} / {cpitch}: one luma and one chroma "
                                 "pitch per call")
            if x < 0 or y < 0 or x + w > W or y + h > H:
                raise ValueError(f"pictures[{i}]: the {w}x{h} frame at ({x}, {y}) leaves the {W}x{H} picture")
            if c420 and (x % 2 or y % 2):
                raise ValueError(f"pictures[{i}]: a {fmt} frame starts at an even (x, y), got ({x}, {y})")
            if c422 and x % 2:
                raise ValueError(f"pictures[{i}]: a {fmt} frame starts at an even x, got ({x}, {y})")
            cx, cy = (x // 2, y // 2) if c420 else (x // 2, y) if c422 else (x, y)
            cs = {"nv12": 2, "p010": 4, "i420": 1, "yuv420p10": 2}.get(fmt, sb)   # chroma bytes per chroma position
            ptrs = [bases[0] + y * P + x * px] + [bases[p] + cy * CP + cx * cs for p in range(1, nplanes)]
            for p, a in enumerate(ptrs):
                if a % 16:
                    raise ValueError(f"pictures[{i}]: the frame at ({x}, {y}) starts plane {p} at an address that is not a "
                                     "multiple of 16 bytes")
            arr[i].plane = (C.c_void_p * 3)(*(ptrs + [None] * (3 - nplanes)))
        desc = OverlayPlanesDesc()
        desc.format = EXPORT_FORMATS[fmt]
        desc.flags = _colour_flags(matrix, full_range, transfer)
        desc.pitch, desc.chroma_pitch = pitch or 0, cpitch or 0
        return s, desc, arr


def _export_desc(fmt, over, background, matrix="bt709", full_range=False, straight=False, transfer=None):
    """the Export descriptor of a format name, the composite flag, an RGB(A) background (pitch and uv_offset 0), the
    Y'CbCr encoding: matrix "bt709" or "bt601", full_range (DESIGN 4.15; the defaults set no flag, and a matrix or range
    on RGBA / BGRA reaches the library's refusal), or matrix "bt2020" with transfer "pq" / "hlg" (DESIGN 4.22), and straight
    alpha (DESIGN 4.19; on a Y'CbCr format it reaches the library's refusal)"""
    if fmt not in EXPORT_FORMATS:
        raise ValueError(f"format {fmt!r}: one of {sorted(EXPORT_FORMATS)}")
    colour = _colour_flags(matrix, full_range, transfer)
    if straight and over:
        raise ValueError("straight and over exclude each other: a composite is opaque")
    desc = Export()
    desc.format = EXPORT_FORMATS[fmt]
    desc.flags = (EXPORT_OVER if over else 0) | (EXPORT_STRAIGHT if straight else 0) | colour
    bg = [int(v) for v in background]
    assert len(bg) in (3, 4), background
    desc.background = (C.c_uint8 * 4)(*bg[:3], 0)
    return desc


def _export_scale(size, crop):
    """the ExportScale of an output size (w, h) and a crop (x, y, w, h) in top-down coordinates (None: the whole frame)"""
    sc = ExportScale()
    sc.src_x, sc.src_y, sc.src_w, sc.src_h = (0, 0, 0, 0) if crop is None else (int(v) for v in crop)
    sc.out_w, sc.out_h = (int(v) for v in size)
    return sc


def _event_handle(ev, stream=None):
    """a cudaEvent_t as an integer (None: none): an integer handle, or a torch.cuda.Event — one that was never recorded is
    created by recording it on `stream` (None: nothing to wait for)"""
    if ev is None or isinstance(ev, int):
        return ev
    if not ev.cuda_event:
        if stream is None:
            return None
        ev.record(stream)
    return ev.cuda_event


class Pipe:
    """live `--pipe NAME[:TYPE]` binds fed with stdin text (glava.c:338-411, render.c:1846-2100)"""

    def __init__(self, pipe_args, paths=None, entry="rc.glsl", requests=None, force_module=None):
        self._L = lib()
        self._h = self._L.glava_b200_pipe_new(_cstr_array(paths), entry.encode() if entry else None, _cstr_array(requests),
                                              force_module.encode() if force_module else None, _cstr_array(list(pipe_args)))
        if not self._h:
            raise GlavaError(self._L.glava_b200_last_error().decode(errors="replace"))
        self.messages = []

    def feed(self, text):
        """-> number of binds that took a new value; parse complaints (reference wording) are appended to .messages"""
        data = text.encode() if isinstance(text, str) else bytes(text)
        n = self._L.glava_b200_pipe_feed(self._h, data, len(data))
        if n < 0:
            raise GlavaError(self._L.glava_b200_last_error().decode(errors="replace"))
        return n

    def params(self):
        p = Params()
        _check(self._L.glava_b200_pipe_params(self._h, C.byref(p)))
        return p

    def binds(self):
        out = {}
        for i in range(self._L.glava_b200_pipe_bind_count(self._h)):
            name, typ, val = C.c_char_p(), C.c_char_p(), (C.c_float * 4)()
            _check(self._L.glava_b200_pipe_bind(self._h, i, C.byref(name), C.byref(typ), val))
            out[name.value.decode()] = (typ.value.decode(), tuple(val))
        return out

    def apply(self, renderer):
        _check(self._L.glava_b200_pipe_apply(self._h, renderer._h))
        _check(self._L.glava_b200_get_params(renderer._h, C.byref(renderer.params)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.glava_b200_pipe_free(self._h)
            self._h = None

    def __enter__(self): return self
    def __exit__(self, *a): self.close()


_pinned = []


def pinned_empty(shape, dtype, device=None):
    """numpy array backed by pinned host memory on the NUMA node of `device` (default: the current CUDA device);
    lives until process exit."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    ptr = lib().glava_b200_host_alloc(nbytes) if device is None else lib().glava_b200_host_alloc_on(nbytes, int(device))
    if not ptr:
        raise GlavaError("pinned allocation failed")
    buf = (C.c_byte * nbytes).from_address(ptr)
    _pinned.append(buf)
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


class Renderer(_StreamState, _StreamStyles, _FrameExport):
    """Batched renderer handle: the role of struct glava_renderer (render.h:8-30)."""

    @property
    def _style_fn(self):
        return self._L.glava_b200_set_stream_styles, self._L.glava_b200_get_stream_styles

    @property
    def _fn(self):
        return self._L.glava_b200_reset_streams, self._L.glava_b200_save_streams, self._L.glava_b200_load_streams

    def __init__(self, params, batch=1, device=0):
        self._L = lib()
        self._h = self._L.glava_b200_new(C.byref(params), int(batch), int(device))
        if not self._h:
            raise GlavaError(self._L.glava_b200_last_error().decode(errors="replace"))
        self.params = Params()
        _check(self._L.glava_b200_get_params(self._h, C.byref(self.params)))
        self.batch = int(batch)
        self.device = int(device)
        self.nsz = int(self._L.glava_b200_spectrum_size(self._h))      # params.n / bufscale: spectrum / texture entries

    # -- rd_update ---------------------------------------------------------------------------------
    def update(self, lb, rb=None, modified=True):
        """lb, rb: host float32 arrays [batch][n] (ring contents oldest-first)."""
        lb = np.ascontiguousarray(lb, dtype=np.float32)
        assert lb.shape == (self.batch, self.params.n), lb.shape
        rp = None
        if rb is not None:
            rb = np.ascontiguousarray(rb, dtype=np.float32)
            assert rb.shape == lb.shape
            rp = rb.ctypes.data
        _check(self._L.glava_b200_update(self._h, lb.ctypes.data, rp, self.params.n, 1 if modified else 0))
        self._after_update()

    def _mask(self, modified):
        m = np.ascontiguousarray(np.asarray(modified) != 0, dtype=np.uint8)
        assert m.shape == (self.batch,), m.shape
        return m

    def update_masked(self, lb, rb, modified):
        """per-stream `modified` flags ([batch] booleans): glava.c:528-537 per stream"""
        lb = np.ascontiguousarray(lb, dtype=np.float32); rb = np.ascontiguousarray(rb, dtype=np.float32)
        assert lb.shape == (self.batch, self.params.n) and rb.shape == lb.shape
        m = self._mask(modified)
        _check(self._L.glava_b200_update_masked(self._h, lb.ctypes.data, rb.ctypes.data, self.params.n, m.ctypes.data))
        self._after_update()

    def update_device_masked(self, d_lb, d_rb, modified):
        m = self._mask(modified)
        _check(self._L.glava_b200_update_device_masked(self._h, d_lb, d_rb, self.params.n, m.ctypes.data))
        self._after_update()

    def update_rings_masked(self, modified):
        m = self._mask(modified)
        _check(self._L.glava_b200_update_rings_masked(self._h, m.ctypes.data))
        self._after_update()

    def _after_update(self):
        if getattr(self, "_resize_pending", False):          # a glava_b200_sizereq was applied by this update
            self._resize_pending = False
            self.refresh_params()

    def reconfigure(self, params):
        """live parameter update (colours, amplify, smoothing...): the `--pipe` analogue"""
        _check(self._L.glava_b200_reconfigure(self._h, C.byref(params)))
        _check(self._L.glava_b200_get_params(self._h, C.byref(self.params)))

    def update_device(self, d_lb, d_rb, modified=True):
        """d_lb, d_rb: integer device addresses of [batch][n] float32 (e.g. torch tensor.data_ptr())."""
        _check(self._L.glava_b200_update_device(self._h, d_lb, d_rb, self.params.n, 1 if modified else 0))
        self._after_update()

    def update_device_after(self, d_lb, d_rb, modified, ready_event):
        """update_device ordered after `ready_event` (a cudaEvent_t handle, e.g. torch.cuda.Event().cuda_event)"""
        _check(self._L.glava_b200_update_device_after(self._h, d_lb, d_rb, self.params.n, 1 if modified else 0, ready_event))
        self._after_update()

    @property
    def input_event(self):
        return self._L.glava_b200_input_event(self._h)

    def ingest_fifo(self, chunks):
        chunks = np.ascontiguousarray(chunks, dtype=np.int16)
        assert chunks.ndim == 2 and chunks.shape[0] == self.batch and chunks.shape[1] % 2 == 0
        _check(self._L.glava_b200_ingest_fifo(self._h, chunks.ctypes.data, chunks.shape[1] // 2))

    def ingest_float(self, chunks):
        """PulseAudio semantics (pulse_input.c:146-174): float samples as they are, [batch][frames*2] interleaved"""
        chunks = np.ascontiguousarray(chunks, dtype=np.float32)
        assert chunks.ndim == 2 and chunks.shape[0] == self.batch and chunks.shape[1] % 2 == 0
        _check(self._L.glava_b200_ingest_float(self._h, chunks.ctypes.data, chunks.shape[1] // 2))

    def update_rings(self, modified=True):
        _check(self._L.glava_b200_update_rings(self._h, 1 if modified else 0))
        self._after_update()

    def set_async_input(self, enable=True):
        _check(self._L.glava_b200_set_async_input(self._h, 1 if enable else 0))

    def wait_input(self):
        _check(self._L.glava_b200_wait_input(self._h))

    def sync(self):
        _check(self._L.glava_b200_sync(self._h))

    # -- outputs -----------------------------------------------------------------------------------
    def readback(self, stream=0, out=None):
        p = self.params
        if out is None:
            out = np.empty((p.h, p.w, 4), dtype=np.uint8)
        _check(self._L.glava_b200_readback(self._h, int(stream), out.ctypes.data))
        return out

    def readback_async(self, stream, out):
        """enqueue the D2H copy of one frame into `out` (pinned uint8 [h][w][4]); valid after sync()"""
        _check(self._L.glava_b200_readback_async(self._h, int(stream), out.ctypes.data))

    def readback_fence(self):
        """order later work on cuda_stream after the read-backs issued so far (their D2H runs on a separate stream)"""
        _check(self._L.glava_b200_readback_fence(self._h))

    def spectrum(self):
        l = np.empty((self.batch, self.nsz), dtype=np.float32); r = np.empty_like(l)
        _check(self._L.glava_b200_spectrum(self._h, l.ctypes.data, r.ctypes.data))
        return l, r

    def textures(self):
        l = np.empty((self.batch, self.nsz), dtype=np.uint16); r = np.empty_like(l)
        _check(self._L.glava_b200_textures(self._h, l.ctypes.data, r.ctypes.data))
        return l, r

    def smooth_pass(self, tex):
        tex = np.ascontiguousarray(tex, dtype=np.uint16)
        assert tex.ndim == 2 and tex.shape[1] == self.nsz
        out = np.empty_like(tex)
        _check(self._L.glava_b200_smooth_pass(self._h, tex.ctypes.data, out.ctypes.data, tex.shape[0]))
        return out

    def transform_smooth(self, planes):
        """transform_smooth (render.c:694-718) on host float32 [count][nsz]; returns the transformed copy"""
        b = np.array(planes, dtype=np.float32, copy=True)
        assert b.ndim == 2 and b.shape[1] == self.nsz
        _check(self._L.glava_b200_transform_smooth(self._h, b.ctypes.data, b.shape[0]))
        return b

    def raster_textures(self, tex_l, tex_r=None):
        tex_l = np.ascontiguousarray(tex_l, dtype=np.uint16)
        assert tex_l.shape == (self.batch, self.nsz)
        rp = None
        if tex_r is not None:
            tex_r = np.ascontiguousarray(tex_r, dtype=np.uint16)
            rp = tex_r.ctypes.data
        _check(self._L.glava_b200_raster_textures(self._h, tex_l.ctypes.data, rp))

    def timeline(self, cap=4096):
        """(spectrum [k][2], raster [m][2]) start/end ms of the timed launches (set_timing(True) first)"""
        out = np.zeros((cap, 2), np.float64); ns, nq = C.c_int(), C.c_int()
        _check(self._L.glava_b200_timeline(self._h, out.ctypes.data, cap, C.byref(ns), C.byref(nq)))
        return out[: ns.value].copy(), out[ns.value: ns.value + nq.value].copy()

    # -- offscreen hand-off (glava_sizereq / glava_wait / glava_tex) ---------------------------------
    def sizereq(self, w, h):
        """resize request, applied at the start of the next update"""
        _check(self._L.glava_b200_sizereq(self._h, int(w), int(h)))
        self._resize_pending = True

    def refresh_params(self):
        _check(self._L.glava_b200_get_params(self._h, C.byref(self.params)))
        return self.params

    def wait_frame(self):
        _check(self._L.glava_b200_wait_frame(self._h))

    @property
    def frame_event(self):
        return self._L.glava_b200_frame_event(self._h)

    def frame_device(self, stream):
        return self._L.glava_b200_frame_device(self._h, int(stream))

    def framebuffer_ipc(self):
        buf = (C.c_ubyte * 64)()
        _check(self._L.glava_b200_framebuffer_ipc(self._h, buf, 64))
        return bytes(buf)

    @property
    def framebuffer_device(self):
        return self._L.glava_b200_framebuffer_device(self._h)

    def export_frames(self, streams, fmt="rgba", over=False, background=(0, 0, 0), out=None, after=None, done=None,
                      matrix="bt709", full_range=False, straight=False, transfer=None):
        """The current frames of `streams` (repeats allowed) top-down in the caller's device memory (glava_b200_export_frames):
        fmt "rgba" / "bgra" ([h, w, 4] per frame; over=True composites over `background` as GLava's window shows it) or
        "nv12" ([h * 3 / 2, w]: Y rows, then interleaved CbCr rows), "p010" (the same as uint16 samples, 10-bit code << 6),
        "i420" / "yuv444" (a tuple of plane views Y [h, w], Cb and Cr [h / 2, w / 2] or [h, w] of one back-to-back
        allocation), "yuv420p10" / "yuv444p10" (the same planes as uint16 samples holding the 10-bit code in their low bits:
        ffmpeg's yuv420p10le / yuv444p10le), "yuv422p" / "yuv422p10" (Y [h, w], Cb and Cr [h, w / 2], uint8 / uint16) or
        "uyvy" ([h, 2 w] uint8, Cb Y0 Cr Y1 per pixel pair), or "yuva420p" / "yuva444p10" (I420's / YUV444P10's planes and an A
        plane [h, w]: (Y, Cb, Cr, A), ffmpeg's yuva420p / yuva444p10le, never composited: the straight colour and the frame's
        alpha, DESIGN 4.19); the other YUV formats are always composited.  straight=True (RGBA / BGRA, not with over): the
        colour un-premultiplied, as PNG and ffmpeg's rgba take it.  out: see _export_plan; None allocates
        [count, ...] of those shapes (rows padded to a multiple of 16 bytes, 32 for I420, YUV420P10, YUV422P and YUV422P10).  Returns out.
        after / done: torch.cuda.Event or cudaEvent_t handles — the export waits for `after` on the device and records
        `done` behind itself.  Left None, the export is ordered after the work already queued on torch's current stream,
        and that stream waits for the export (the tensors can be used right away).
        matrix ("bt709" / "bt601") and full_range: the Y'CbCr encoding of every YUV format (DESIGN 4.15; the
        default is BT.709 limited range; matrix="bt601", full_range=True is JPEG's).  matrix="bt2020" with transfer="pq" or
        "hlg": BT.2020 HDR10 / HLG limited range on p010, yuv420p10, yuv444p10 and yuv422p10, SDR graphics white at 203 cd/m^2
        (DESIGN 4.22)."""
        s, desc, dst, result = self._export_plan(streams, fmt, over, background, out, lambda stream: self.device, None, matrix,
                                                 full_range, straight, transfer)
        self._ordered(lambda a, d: self._L.glava_b200_export_frames(self._h, s.ctypes.data, s.shape[0], dst, C.byref(desc), a, d),
                      after, done)
        return result

    def _ordered(self, call, after, done):
        """call(after_event, done_event) on the handle's stream, ordered against torch's current stream as export_frames
        describes"""
        import torch
        dev = torch.device("cuda", self.device)
        cur = torch.cuda.current_stream(dev)
        own = torch.cuda.ExternalStream(self.cuda_stream, device=dev)
        if after is None:
            own.wait_stream(cur)
        _check(call(_event_handle(after), _event_handle(done, cur)))
        if done is None:
            cur.wait_stream(own)

    def export_scaled(self, streams, size, crop=None, fmt="rgba", over=False, background=(0, 0, 0), out=None, after=None,
                      done=None, matrix="bt709", full_range=False, straight=False, transfer=None):
        """export_frames of a source rectangle shrunk to size = (w, h) by the exact area average (glava_b200_export_scaled):
        crop = (x, y, w, h) in top-down coordinates (y = 0 is the top row), None: the whole frame.  Downscale only; NV12,
        I420, P010 and YUV420P10 need an even w and h, YUV422P, YUV422P10 and UYVY an even w.  Shapes, out, after, done, matrix, full_range and transfer as export_frames, with the output
        size in place of the frame's; straight as export_frames (the stored channels averaged, then un-premultiplied)."""
        s, desc, dst, result = self._export_plan(streams, fmt, over, background, out, lambda stream: self.device, size, matrix,
                                                 full_range, straight, transfer)
        sc = _export_scale(size, crop)
        self._ordered(lambda a, d: self._L.glava_b200_export_scaled(self._h, s.ctypes.data, s.shape[0], dst, None, C.byref(desc),
                                                                    C.byref(sc), a, d), after, done)
        return result

    def export_ladder(self, streams, rungs, out=None, after=None, done=None):
        """Several sizes of each frame in one launch that reads each source row about once (glava_b200_export_ladder), for
        an encoder ladder: rungs = [dict(size=(w, h) or None for the frame's, crop=None, fmt="nv12", over=False,
        background=(0, 0, 0), matrix="bt709", full_range=False, straight=False, transfer=None), ...], at most LADDER_MAX; rungs may
        mix encodings, HDR and SDR included.  Rung j is exactly export_scaled(streams, **rungs[j]) at this
        point in call order.  out: None or one entry per rung in any form export_scaled takes.  Returns one result per rung,
        shaped as export_scaled returns it; after / done and the ordering against torch's current stream as export_frames."""
        s, arr, n, dst, results = self._ladder_plan(streams, rungs, out, lambda stream: self.device)
        self._ordered(lambda a, d: self._L.glava_b200_export_ladder(self._h, s.ctypes.data, s.shape[0], arr, n, dst, None, a, d),
                      after, done)
        return results

    def overlay_frames(self, streams, images, at=None, fmt="nv12", after=None, done=None, matrix="bt709", full_range=False,
                       opacity=None, size=None, crop=None):
        """The current frames of `streams` composited in place onto the caller's images (glava_b200_overlay_frames): under
        native opacity premultiplied "over" the image's pixels, blended in Y'CbCr for NV12; under any other opacity the
        opaque bytes export_frames writes.  images and at: see _overlay_plan; rectangles of one call must not overlap.
        after / done and the ordering against torch's current stream as export_frames.  matrix / full_range: the encoding
        of NV12 pictures, which the blend works in (DESIGN 4.15).  opacity: None, or one float in [0, 1] for every entry or
        one per entry, each frame composited at that strength (glava_b200_overlay_frames_opacity, DESIGN 4.20; under
        any other opacity than native the opaque frame is faded over the image).  size / crop: None, or the frame shrunk
        to size = (w, h) from crop = (x, y, w, h) as export_scaled takes them, composited into a w x h rectangle
        (glava_b200_overlay_scaled, DESIGN 4.21).  Returns images."""
        rect, sc = self._overlay_scale(size, crop)
        s, desc, dst, uv = self._overlay_plan(streams, images, at, fmt, matrix, full_range, rect)
        k = self._opacity(opacity, s.shape[0])
        if sc is not None:
            pd, arr = self._frames_pictures(desc, dst, uv, s.shape[0])
            self._ordered(lambda a, d: self._L.glava_b200_overlay_scaled(self._h, s.ctypes.data, s.shape[0], arr, C.byref(pd),
                                                                         C.byref(sc), None if k is None else k.ctypes.data,
                                                                         a, d), after, done)
        elif k is None:
            self._ordered(lambda a, d: self._L.glava_b200_overlay_frames(self._h, s.ctypes.data, s.shape[0], dst, uv, C.byref(desc),
                                                                         a, d), after, done)
        else:
            self._ordered(lambda a, d: self._L.glava_b200_overlay_frames_opacity(self._h, s.ctypes.data, s.shape[0], dst, uv,
                                                                                 C.byref(desc), k.ctypes.data, a, d), after, done)
        return images

    def overlay_planes(self, streams, pictures, at=None, fmt="i420", matrix="bt709", full_range=False, after=None, done=None,
                       opacity=None, size=None, crop=None, transfer=None):
        """The current frames of `streams` composited in place onto decoded pictures, one tensor per plane
        (glava_b200_overlay_planes): NV12, I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, YUV422P10 or UYVY, the planes of each picture at their
        own addresses with one luma and one chroma pitch per call — ffmpeg's AVFrame planes, NVDEC surfaces, or what
        export_frames returns.  Native opacity blends in Y'CbCr in the picture's encoding (matrix / full_range) as
        overlay_frames blends NV12; any other opacity writes export_frames' bytes.  pictures and at: see _planes_plan;
        rectangles of one call must not overlap in any plane.  after / done and the ordering against torch's current
        stream as export_frames.  opacity: as overlay_frames (glava_b200_overlay_planes_opacity).  size / crop: as
        overlay_frames (glava_b200_overlay_scaled).  matrix="bt2020" with transfer="pq" / "hlg": an HDR picture (p010,
        yuv420p10, yuv444p10, yuv422p10), the graphics blended at 203 cd/m^2 (DESIGN 4.22).  Returns pictures."""
        rect, sc = self._overlay_scale(size, crop)
        s, desc, arr = self._planes_plan(streams, pictures, at, fmt, matrix, full_range, rect, transfer)
        k = self._opacity(opacity, s.shape[0])
        if sc is not None:
            self._ordered(lambda a, d: self._L.glava_b200_overlay_scaled(self._h, s.ctypes.data, s.shape[0], arr, C.byref(desc),
                                                                         C.byref(sc), None if k is None else k.ctypes.data,
                                                                         a, d), after, done)
        elif k is None:
            self._ordered(lambda a, d: self._L.glava_b200_overlay_planes(self._h, s.ctypes.data, s.shape[0], arr, C.byref(desc), a, d),
                          after, done)
        else:
            self._ordered(lambda a, d: self._L.glava_b200_overlay_planes_opacity(self._h, s.ctypes.data, s.shape[0], arr,
                                                                                 C.byref(desc), k.ctypes.data, a, d), after, done)
        return pictures

    def export_mosaic(self, streams, cols, tile, fmt="nv12", background=(0, 0, 0), out=None, matrix="bt709", full_range=False,
                      transfer=None):
        """The frames of `streams` shrunk to tile = (w, h) and laid out row-major, `cols` tiles per row, in one picture, by
        one export_scaled call with a destination and a chroma destination per tile.  W = cols * w, H = rows * h; returns
        [H * 3 / 2, W] for NV12 (uint8) and P010 (uint16), Y rows then CbCr rows, the plane views (Y, Cb, Cr) for I420 and
        YUV444 (uint8) and YUV420P10 and YUV444P10 (uint16), the same for YUV422P (uint8) and YUV422P10 (uint16), [H, 2 W]
        for UYVY, or [H, W, 4]: one surface to hand to an encoder.  Tiles start at multiples of 16 bytes in every plane, so w
        is a multiple of 16 (NV12, YUV444, YUV420P10, YUV422P10), 32 (I420, YUV422P), 8 (P010, YUV444P10, UYVY) or 4 (RGBA /
        BGRA).  out: a CUDA tensor [rows, pitch] whose rows hold the picture's row bytes, rows as
        _export_layout gives them for W x H (planar formats: the chroma planes back to back from row H); tiles past the last
        stream keep its bytes (out None: black).  Ordered against torch's current stream as export_frames without events.
        matrix / full_range / transfer as export_frames (black: Y 0 in full range, 64 in limited range and HDR)."""
        import torch
        s = np.ascontiguousarray(np.asarray(streams, dtype=np.int64).reshape(-1), dtype=np.int32)
        count, cols = int(s.shape[0]), int(cols)
        tw, th = (int(v) for v in tile)
        if count < 1 or cols < 1:
            raise ValueError("export_mosaic: at least one stream and one column")
        if fmt in ALPHA_FORMATS:
            raise ValueError(f"export_mosaic: format {fmt!r}: a mosaic is one opaque picture, it takes no alpha format")
        desc = _export_desc(fmt, False, background, matrix, full_range, transfer=transfer)
        W, H = cols * tw, (count + cols - 1) // cols * th
        rows, row_bytes, align = _export_layout(fmt, W, H)
        px = {"rgba": 4, "bgra": 4, "uyvy": 2}.get(fmt, 2 if fmt in WIDE_FORMATS else 1)
        if out is None:
            base = torch.empty((rows, (row_bytes + align - 1) // align * align), dtype=torch.uint8, device=f"cuda:{self.device}")
            if count % cols:                                  # black where no stream lands
                if fmt == "p010":
                    base.view(torch.uint16)[:H].fill_(0 if full_range else 64 << 6)
                    base.view(torch.uint16)[H:].fill_(512 << 6)
                elif fmt in ("yuv420p10", "yuv444p10", "yuv422p10"):
                    base.view(torch.uint16)[:H].fill_(0 if full_range else 64)
                    base.view(torch.uint16)[H:].fill_(512)
                elif fmt == "uyvy":                           # Cb, Y, Cr, Y: 128, 16 (full range 128, 0) per pixel
                    base.view(torch.uint16).fill_(128 | (0 if full_range else 16) << 8)
                elif fmt in ("rgba", "bgra"):
                    base.fill_(0)
                else:
                    base[:H].fill_(0 if full_range else 16)
                    base[H:].fill_(128)
            result = _export_views(fmt, base, W, H)
        else:
            dtypes = (torch.uint8, torch.uint16) if fmt in WIDE_FORMATS else (torch.uint8,)
            if (out.dtype not in dtypes or not out.is_cuda or out.dim() != 2 or out.shape[0] != rows or out.stride(1) != 1
                    or out.shape[1] * out.element_size() < row_bytes):
                raise ValueError(f"out: a uint8 CUDA tensor [{rows}, >= {row_bytes}] with contiguous rows")
            base = result = out
        pitch, ptr = base.stride(0) * base.element_size(), base.data_ptr()
        dst = (C.c_void_p * count)(*[ptr + (i // cols) * th * pitch + (i % cols) * tw * px for i in range(count)])
        if fmt in ("nv12", "p010"):
            uv = [ptr + (H + (i // cols) * (th // 2)) * pitch + (i % cols) * tw * px for i in range(count)]
        elif fmt in ("i420", "yuv420p10"):                    # Cr one whole chroma plane past Cb
            uv = [ptr + H * pitch + (i // cols) * (th // 2) * (pitch // 2) + (i % cols) * (tw // 2) * px for i in range(count)]
            desc.uv_offset = (pitch // 2) * (H // 2)
        elif fmt in ("yuv422p", "yuv422p10"):                 # chroma rows pitch / 2 apart, Cr one plane past Cb
            uv = [ptr + H * pitch + (i // cols) * th * (pitch // 2) + (i % cols) * (tw // 2) * px for i in range(count)]
            desc.uv_offset = (pitch // 2) * H
        elif fmt in ("yuv444", "yuv444p10"):
            uv = [ptr + (H + (i // cols) * th) * pitch + (i % cols) * tw * px for i in range(count)]
            desc.uv_offset = pitch * H
        else:
            uv = None
        uv = (C.c_void_p * count)(*uv) if uv else None
        desc.pitch = pitch
        sc = _export_scale(tile, None)
        self._ordered(lambda a, d: self._L.glava_b200_export_scaled(self._h, s.ctypes.data, count, dst, uv, C.byref(desc),
                                                                    C.byref(sc), a, d), None, None)
        return result

    @property
    def cuda_stream(self):
        return self._L.glava_b200_cuda_stream(self._h)

    @property
    def launch_count(self):
        return int(self._L.glava_b200_launch_count(self._h))

    def set_timing(self, enable=True):
        _check(self._L.glava_b200_set_timing(self._h, 1 if enable else 0))

    def kernel_times(self):
        """-> dict(spectrum_ms, spectrum_launches, raster_ms, raster_launches) since set_timing(True)"""
        s, q = C.c_double(), C.c_double()
        ns, nq = C.c_int(), C.c_int()
        _check(self._L.glava_b200_kernel_times(self._h, C.byref(s), C.byref(ns), C.byref(q), C.byref(nq)))
        return dict(spectrum_ms=s.value, spectrum_launches=ns.value, raster_ms=q.value, raster_launches=nq.value)

    # -- rd_destroy --------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._L.glava_b200_destroy(self._h)
            self._h = None

    def __enter__(self): return self
    def __exit__(self, *a): self.close()
    def __del__(self):
        try: self.close()
        except Exception: pass


class ShardedRenderer(_StreamState, _StreamStyles, _FrameExport):
    """One handle for a batch spread over several GPUs of a node (glava_b200_new_sharded): contiguous stream blocks, one
    worker thread per device, no inter-device traffic.  devices: list of CUDA ordinals (may repeat), or None = all visible.
    reset_streams / save_streams / load_streams take global stream indices."""

    @property
    def _style_fn(self):
        return self._L.glava_b200_sharded_set_stream_styles, self._L.glava_b200_sharded_get_stream_styles

    @property
    def _fn(self):
        return (self._L.glava_b200_sharded_reset_streams, self._L.glava_b200_sharded_save_streams,
                self._L.glava_b200_sharded_load_streams)

    def __init__(self, params, batch, devices=None):
        self._L = lib()
        if devices is None:
            self._h = self._L.glava_b200_new_sharded(C.byref(params), int(batch), 0)
        else:
            arr = (C.c_int * len(devices))(*[int(d) for d in devices])
            self._h = self._L.glava_b200_new_sharded_devices(C.byref(params), int(batch), arr, len(devices))
        if not self._h:
            raise GlavaError(self._L.glava_b200_last_error().decode(errors="replace"))
        self.params = params.copy()
        self.batch = int(batch)

    @property
    def shards(self):
        """[(device, first_stream, count)]"""
        out = []
        for k in range(self._L.glava_b200_sharded_shards(self._h)):
            d, f, c = C.c_int(), C.c_int(), C.c_int()
            self._L.glava_b200_sharded_shard(self._h, k, C.byref(d), C.byref(f), C.byref(c))
            out.append((d.value, f.value, c.value))
        return out

    def update(self, lb, rb, modified=None):
        lb = np.ascontiguousarray(lb, dtype=np.float32); rb = np.ascontiguousarray(rb, dtype=np.float32)
        assert lb.shape == (self.batch, self.params.n) and rb.shape == lb.shape
        m = None
        if modified is not None:
            m = np.ascontiguousarray(np.asarray(modified) != 0, dtype=np.uint8)
            assert m.shape == (self.batch,)
        _check(self._L.glava_b200_sharded_update(self._h, lb.ctypes.data, rb.ctypes.data, self.params.n, m.ctypes.data if m is not None else None))

    def rerender(self):
        _check(self._L.glava_b200_sharded_rerender(self._h))

    def ingest_fifo(self, chunks):
        chunks = np.ascontiguousarray(chunks, dtype=np.int16)
        assert chunks.ndim == 2 and chunks.shape[0] == self.batch and chunks.shape[1] % 2 == 0
        _check(self._L.glava_b200_sharded_ingest_fifo(self._h, chunks.ctypes.data, chunks.shape[1] // 2))

    def sync(self):
        _check(self._L.glava_b200_sharded_sync(self._h))

    def readback(self, stream, out=None):
        p = self.params
        if out is None:
            out = np.empty((p.h, p.w, 4), dtype=np.uint8)
        _check(self._L.glava_b200_sharded_readback(self._h, int(stream), out.ctypes.data))
        return out

    def textures(self):
        n = self.params.n // max(self.params.bufscale, 1)
        l = np.empty((self.batch, n), dtype=np.uint16); r = np.empty_like(l)
        _check(self._L.glava_b200_sharded_textures(self._h, l.ctypes.data, r.ctypes.data))
        return l, r

    def export_frames(self, streams, fmt="rgba", over=False, background=(0, 0, 0), out=None, matrix="bt709", full_range=False,
                      straight=False, transfer=None):
        """Renderer.export_frames with global stream indices (glava_b200_sharded_export_frames): each destination on the
        device of the shard that owns its stream (out None: one tensor when every listed stream lives on one device, else
        a list of per-frame tensors).  Work queued on torch's current streams of those devices is waited for first; the
        frames are complete after sync().  matrix / full_range / straight / transfer as Renderer.export_frames."""
        import torch
        device_of = self._device_of()
        s, desc, dst, result = self._export_plan(streams, fmt, over, background, out, device_of, None, matrix, full_range, straight,
                                                 transfer)
        for d in sorted({device_of(int(x)) for x in s}):
            torch.cuda.current_stream(d).synchronize()
        _check(self._L.glava_b200_sharded_export_frames(self._h, s.ctypes.data, s.shape[0], dst, C.byref(desc)))
        return result

    def export_scaled(self, streams, size, crop=None, fmt="rgba", over=False, background=(0, 0, 0), out=None, matrix="bt709",
                      full_range=False, straight=False, transfer=None):
        """Renderer.export_scaled with global stream indices (glava_b200_sharded_export_scaled), destinations placed as
        export_frames places them; the frames are complete after sync().  matrix / full_range / straight as
        Renderer.export_frames."""
        import torch
        device_of = self._device_of()
        s, desc, dst, result = self._export_plan(streams, fmt, over, background, out, device_of, size, matrix, full_range, straight,
                                                 transfer)
        sc = _export_scale(size, crop)
        for d in sorted({device_of(int(x)) for x in s}):
            torch.cuda.current_stream(d).synchronize()
        _check(self._L.glava_b200_sharded_export_scaled(self._h, s.ctypes.data, s.shape[0], dst, None, C.byref(desc), C.byref(sc)))
        return result

    def export_ladder(self, streams, rungs, out=None):
        """Renderer.export_ladder with global stream indices (glava_b200_sharded_export_ladder), destinations placed as
        export_frames places them; the frames are complete after sync()."""
        import torch
        device_of = self._device_of()
        s, arr, n, dst, results = self._ladder_plan(streams, rungs, out, device_of)
        for d in sorted({device_of(int(x)) for x in s}):
            torch.cuda.current_stream(d).synchronize()
        _check(self._L.glava_b200_sharded_export_ladder(self._h, s.ctypes.data, s.shape[0], arr, n, dst, None))
        return results

    def overlay_frames(self, streams, images, at=None, fmt="nv12", matrix="bt709", full_range=False, opacity=None, size=None,
                       crop=None):
        """Renderer.overlay_frames with global stream indices (glava_b200_sharded_overlay_frames), each image on the device
        of the shard that owns its stream.  Work queued on torch's current streams of those devices is waited for first;
        the images are complete after sync().  matrix / full_range / opacity / size / crop as Renderer.overlay_frames."""
        import torch
        device_of = self._device_of()
        rect, sc = self._overlay_scale(size, crop)
        s, desc, dst, uv = self._overlay_plan(streams, images, at, fmt, matrix, full_range, rect)
        k = self._opacity(opacity, s.shape[0])
        for d in sorted({device_of(int(x)) for x in s if 0 <= int(x) < self.batch}):
            torch.cuda.current_stream(d).synchronize()
        if sc is not None:
            pd, arr = self._frames_pictures(desc, dst, uv, s.shape[0])
            _check(self._L.glava_b200_sharded_overlay_scaled(self._h, s.ctypes.data, s.shape[0], arr, C.byref(pd), C.byref(sc),
                                                             None if k is None else k.ctypes.data))
        elif k is None:
            _check(self._L.glava_b200_sharded_overlay_frames(self._h, s.ctypes.data, s.shape[0], dst, uv, C.byref(desc)))
        else:
            _check(self._L.glava_b200_sharded_overlay_frames_opacity(self._h, s.ctypes.data, s.shape[0], dst, uv, C.byref(desc),
                                                                     k.ctypes.data))
        return images

    def overlay_planes(self, streams, pictures, at=None, fmt="i420", matrix="bt709", full_range=False, opacity=None, size=None,
                       crop=None, transfer=None):
        """Renderer.overlay_planes with global stream indices (glava_b200_sharded_overlay_planes), each picture on the device
        of the shard that owns its stream.  Work queued on torch's current streams of those devices is waited for first;
        the pictures are complete after sync().  opacity / size / crop as Renderer.overlay_frames."""
        import torch
        device_of = self._device_of()
        rect, sc = self._overlay_scale(size, crop)
        s, desc, arr = self._planes_plan(streams, pictures, at, fmt, matrix, full_range, rect, transfer)
        k = self._opacity(opacity, s.shape[0])
        for d in sorted({device_of(int(x)) for x in s if 0 <= int(x) < self.batch}):
            torch.cuda.current_stream(d).synchronize()
        if sc is not None:
            _check(self._L.glava_b200_sharded_overlay_scaled(self._h, s.ctypes.data, s.shape[0], arr, C.byref(desc), C.byref(sc),
                                                             None if k is None else k.ctypes.data))
        elif k is None:
            _check(self._L.glava_b200_sharded_overlay_planes(self._h, s.ctypes.data, s.shape[0], arr, C.byref(desc)))
        else:
            _check(self._L.glava_b200_sharded_overlay_planes_opacity(self._h, s.ctypes.data, s.shape[0], arr, C.byref(desc),
                                                                     k.ctypes.data))
        return pictures

    def _device_of(self):
        """stream -> the CUDA device of the shard that owns it"""
        shards = self.shards

        def device_of(stream):
            for d, first, cnt in shards:
                if first <= stream < first + cnt:
                    return d
            return shards[0][0]
        return device_of

    def close(self):
        if getattr(self, "_h", None):
            self._L.glava_b200_sharded_destroy(self._h)
            self._h = None

    def __enter__(self): return self
    def __exit__(self, *a): self.close()
    def __del__(self):
        try: self.close()
        except Exception: pass
