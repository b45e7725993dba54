"""glava_b200 — GPU-native GLava hot path (PCM -> spectrum -> pixels).

Thin ctypes binding over the C ABI in ``include/glava_b200.h`` (``libglava_b200.so``,
hand-written sm_90a CUDA).  The Python layer only marshals pointers; it mirrors the
reference's renderer interface (glava/render.h:53-60):

    rd_new      -> Renderer(params, batch, device)
    rd_update   -> Renderer.update(lb, rb, modified)
    rd_destroy  -> Renderer.close()
    (a batch over several GPUs of a node: ShardedRenderer, glava_b200_new_sharded)

There is no CPU fallback: constructing a Renderer without the CUDA library or without a GPU
raises.
"""
from .api import (Params, Color, Renderer, GlavaError, default_params, load_config, lib, lib_path,
                  MODULES, pinned_empty, Pipe, ShardedRenderer, stream_state_bytes, STATE_HEADER_BYTES,
                  StreamStyle, stream_style, style_params, STYLE_AMPLIFY, STYLE_FG, STYLE_BG,
                  Export, ExportScale, ExportRung, LADDER_MAX, EXPORT_RGBA, EXPORT_BGRA, EXPORT_NV12, EXPORT_I420,
                  EXPORT_YUV444, EXPORT_P010, EXPORT_YUV420P10, EXPORT_YUV444P10, EXPORT_YUV422P, EXPORT_YUV422P10,
                  EXPORT_UYVY, EXPORT_YUVA420P, EXPORT_YUVA444P10, EXPORT_OVER, EXPORT_STRAIGHT, EXPORT_FULL_RANGE,
                  EXPORT_BT601, EXPORT_PQ, EXPORT_HLG, Picture, OverlayPlanesDesc, PLANES_FORMATS)
from . import audio
from .synth import synth_pcm_int16, fifo_to_float, StreamRings

__all__ = ["audio", "Params", "Color", "Renderer", "GlavaError", "default_params", "load_config", "lib",
           "lib_path", "MODULES", "pinned_empty", "Pipe", "ShardedRenderer", "stream_state_bytes", "STATE_HEADER_BYTES",
           "StreamStyle", "stream_style", "style_params", "STYLE_AMPLIFY", "STYLE_FG", "STYLE_BG",
           "Export", "ExportScale", "ExportRung", "LADDER_MAX", "EXPORT_RGBA", "EXPORT_BGRA", "EXPORT_NV12", "EXPORT_I420",
           "EXPORT_YUV444", "EXPORT_P010", "EXPORT_YUV420P10", "EXPORT_YUV444P10", "EXPORT_YUV422P",
           "EXPORT_YUV422P10", "EXPORT_UYVY", "EXPORT_YUVA420P", "EXPORT_YUVA444P10", "EXPORT_OVER", "EXPORT_STRAIGHT",
           "EXPORT_FULL_RANGE", "EXPORT_BT601", "EXPORT_PQ", "EXPORT_HLG",
           "Picture", "OverlayPlanesDesc", "PLANES_FORMATS", "synth_pcm_int16",
           "fifo_to_float", "StreamRings"]
