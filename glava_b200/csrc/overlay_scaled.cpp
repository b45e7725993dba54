// overlay_scaled.cpp — the host half of glava_b200_overlay_scaled (DESIGN 4.21): the overlay of a downscaled, cropped frame.
// Its checks are export_scaled's rectangle and overlay_planes' checks against the output size (overlay_planes.cpp, RGBA / BGRA
// taken as one plane); the whole frame at its own size runs the plain overlay's host path and kernels, any other rectangle fills
// one list and launches overlay_scaled_kernel (export_kernels.cu) through export_list.h's enqueue.  Kept apart from
// overlay_planes.cpp so that it builds and links without this launcher.
#include "internal.h"
#include "export_core.h"
#include "export_list.h"

#include <cuda_runtime.h>

#include <vector>

namespace glb {

// The overlay of export_scaled's picture of each frame: the rectangle first (as export_scaled's), then overlay_planes' checks
// against its out_w x out_h output, RGBA / BGRA taken as one plane.
int scaled_overlay_check(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                         const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                         glava_b200_export_scale* q, const char* who) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    const int rc = scale_check(v.w, v.h, scale, q, who);
    return rc ? rc : planes_check(r, streams, count, pics, desc, who, q);
}

int scaled_overlay_run(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                       const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale, const uint8_t* opacity,
                       void* after_event, void* done_event, const char* who) {
    clear_error();
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_export_scale q;
    int rc = scaled_overlay_check(r, streams, count, pics, desc, scale, &q, who);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    const size_t fb_bytes = (size_t) v.slots * (size_t) v.h * (size_t) v.w * 4;
    if ((rc = planes_geometry_check(q.out_w, q.out_h, count, pics, *desc, &v.fb, &fb_bytes, 1, who, true)) != 0) return rc;
    const bool packed = desc->format == GLAVA_B200_EXPORT_RGBA || desc->format == GLAVA_B200_EXPORT_BGRA;
    // the whole frame at its own size is the plain overlay (or its fade), whose kernels it runs, as the ladder's whole rungs
    if (!q.src_x && !q.src_y && q.src_w == v.w && q.src_h == v.h && q.out_w == v.w && q.out_h == v.h) {
        if (!packed) return planes_run(r, streams, count, pics, desc, after_event, done_event, who, opacity);
        std::vector<void*> dst((size_t) count);
        for (int i = 0; i < count; ++i) dst[(size_t) i] = pics[i].plane[0];
        glava_b200_export d = {};
        d.format = desc->format; d.pitch = desc->pitch;
        return export_run(ExportKind::overlay, r, streams, count, dst.data(), nullptr, &d, nullptr, after_event, done_event,
                          opacity, who);
    }
    CU(cudaSetDevice(v.device));
    // K in each entry's pad word, 255 where opacity is null; K = 0 entries are left out of the list (DESIGN 4.20)
    ExportList* L = nullptr;
    size_t bytes = 0;
    if ((rc = planes_list(v, streams, count, pics, opacity, 255, &L, &bytes)) != 0) return rc;
    count = (int) (bytes / sizeof(OverlayPlanesEntry));
    return list_enqueue(v, L, bytes, after_event, done_event, [&](const void* d_list) {
        OverlayScaledArgs a = {};
        a.fb = v.fb;
        a.marks = v.mark_key ? v.marks : nullptr;           // as export.cpp's common_args
        a.mark_rows = v.mark_key >> 2;
        a.list = static_cast<const OverlayPlanesEntry*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
        a.format = desc->format;
        a.native = v.native;
        a.pitch = desc->pitch; a.chroma_pitch = desc->chroma_pitch;
        a.src_x = q.src_x; a.src_y = q.src_y; a.src_w = q.src_w; a.src_h = q.src_h; a.out_w = q.out_w; a.out_h = q.out_h;
        const ExportRecip rcp = export_recip((uint64_t) q.src_w * (uint64_t) q.src_h);
        a.div_mul = rcp.mul; a.div_shift = rcp.shift;
        a.enc = export_enc(desc->flags);
        return launch_overlay_scaled(a, v.stream);
    });
}

}  // namespace glb

extern "C" int glava_b200_overlay_scaled(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                                         const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                                         const uint8_t* opacity, void* after_event, void* done_event) {
    return glb::scaled_overlay_run(r, streams, count, pics, desc, scale, opacity, after_event, done_event, "glava_b200_overlay_scaled");
}
