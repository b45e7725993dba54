// overlay_planes.cpp — the host half of glava_b200_overlay_planes (DESIGN 4.17, 4.18): the overlay onto decoded pictures, whose
// planes each have their own pointer and whose luma and chroma rows have their own pitches.  Its checks, the overlap test
// of rectangles with two pitches, the list fill and one launch of overlay_planes_kernel (export_kernels.cu) through
// export_list.h's enqueue.  Kept apart from export.cpp so that the other exports build and link without this launcher.
#include "internal.h"
#include "export_core.h"
#include "export_list.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <vector>

namespace glb {

namespace {

const char* planes_format_name(int format) {
    switch (format) {
    case GLAVA_B200_EXPORT_NV12: return "NV12";
    case GLAVA_B200_EXPORT_I420: return "I420";
    case GLAVA_B200_EXPORT_YUV444: return "YUV444";
    case GLAVA_B200_EXPORT_P010: return "P010";
    case GLAVA_B200_EXPORT_YUV420P10: return "YUV420P10";
    case GLAVA_B200_EXPORT_YUV444P10: return "YUV444P10";
    case GLAVA_B200_EXPORT_YUV422P: return "YUV422P";
    case GLAVA_B200_EXPORT_YUV422P10: return "YUV422P10";
    case GLAVA_B200_EXPORT_UYVY: return "UYVY";
    case GLAVA_B200_EXPORT_RGBA: return "RGBA";             // the scaled overlay's (DESIGN 4.21)
    case GLAVA_B200_EXPORT_BGRA: return "BGRA";
    default: return nullptr;
    }
}

// plane p of a picture with `planes` planes
const char* plane_name(int planes, int p) { return p == 0 ? "Y" : p == 2 ? "Cr" : planes == 3 ? "Cb" : "CbCr"; }

}  // namespace

int planes_geometry(int w, int h, const glava_b200_overlay_planes_desc& d, PlanesGeom* g, const char* who, bool rgba) {
    const int fmt = d.format;
    const bool packed = fmt == GLAVA_B200_EXPORT_RGBA || fmt == GLAVA_B200_EXPORT_BGRA;
    if (packed && !rgba)
        return fail(GLAVA_B200_EINVAL, "%s: format %s: RGBA and BGRA images go to glava_b200_overlay_frames", who,
                    fmt == GLAVA_B200_EXPORT_RGBA ? "RGBA" : "BGRA");
    if (export_yuva(fmt))                                   // DESIGN 4.19: a transparent layer is exported, not blended onto
        return fail(GLAVA_B200_EINVAL, "%s: format %s: the overlay writes no alpha plane", who,
                    fmt == GLAVA_B200_EXPORT_YUVA420P ? "YUVA420P" : "YUVA444P10");
    const char* name = planes_format_name(fmt);
    if (!name) return fail(GLAVA_B200_EINVAL, "%s: unknown format %d", who, fmt);
    const uint32_t colour = GLAVA_B200_EXPORT_FULL_RANGE | GLAVA_B200_EXPORT_BT601;
    const uint32_t hdr = GLAVA_B200_EXPORT_PQ | GLAVA_B200_EXPORT_HLG;   // the picture's HDR encoding (DESIGN 4.22)
    if (d.flags & GLAVA_B200_EXPORT_STRAIGHT)
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_STRAIGHT is for the exports; the overlay composites", who, d.flags);
    if (d.flags & hdr) {
        const int rc = hdr_flags_check(fmt, d.flags, who);
        if (rc) return rc;
    }
    if (d.flags & ~(colour | hdr))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: the overlay takes none but EXPORT_FULL_RANGE and EXPORT_BT601", who, d.flags);
    if (packed && (d.flags & colour))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: %s has no matrix or range (EXPORT_FULL_RANGE and EXPORT_BT601 are for the "
                    "Y'CbCr formats)", who, d.flags, name);
    const bool c420 = export_420(fmt), uyvy = fmt == GLAVA_B200_EXPORT_UYVY || packed;   // RGBA / BGRA: one plane, as UYVY
    const bool wide = fmt == GLAVA_B200_EXPORT_P010 || export_p10(fmt) || fmt == GLAVA_B200_EXPORT_YUV422P10 || uyvy;
    if (c420 && ((w | h) & 1))
        return fail(GLAVA_B200_EINVAL, "%s: %s needs an even width and height, the frame is %dx%d", who, name, w, h);
    if (export_422(fmt) && (w & 1))
        return fail(GLAVA_B200_EINVAL, "%s: %s needs an even width, the frame is %dx%d", who, name, w, h);
    g->planes = uyvy ? 1 : export_planar(fmt) ? 3 : 2;
    g->luma_row = (size_t) w * (packed ? 4 : wide ? 2 : 1);   // UYVY: its one plane, 2 bytes per pixel
    g->chroma_row = fmt == GLAVA_B200_EXPORT_I420 || fmt == GLAVA_B200_EXPORT_YUV422P ? (size_t) w / 2
                    : fmt == GLAVA_B200_EXPORT_P010 || fmt == GLAVA_B200_EXPORT_YUV444P10 ? (size_t) w * 2
                    : uyvy ? 0 : (size_t) w;
    g->chroma_rows = c420 ? h / 2 : h;
    if (d.pitch % 16 || d.pitch < g->luma_row)
        return fail(GLAVA_B200_EINVAL, "%s: pitch %zu must be a multiple of 16 and at least %zu", who, d.pitch, g->luma_row);
    if (uyvy) {
        if (d.chroma_pitch)
            return fail(GLAVA_B200_EINVAL, "%s: %s chroma_pitch %zu must be 0: %s has no chroma plane", who, name, d.chroma_pitch, name);
        return 0;
    }
    if (d.chroma_pitch % 16 || d.chroma_pitch < g->chroma_row)
        return fail(GLAVA_B200_EINVAL, "%s: %s chroma_pitch %zu must be a multiple of 16 and at least %zu", who, name, d.chroma_pitch,
                    g->chroma_row);
    return 0;
}

int planes_check(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                 const glava_b200_overlay_planes_desc* desc, const char* who, const glava_b200_export_scale* q) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    PlanesGeom g;
    int rc = q ? planes_geometry(q->out_w, q->out_h, *desc, &g, who, true) : planes_geometry(v.w, v.h, *desc, &g, who);
    if (rc) return rc;
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !pics) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    char name[32];
    for (int i = 0; i < count; ++i) {
        if (streams[i] < 0 || streams[i] >= v.batch)
            return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, streams[i], v.batch);
        for (int p = 0; p < g.planes; ++p) {
            snprintf(name, sizeof(name), "pics[%d].plane", i);
            if ((rc = dst_check(v, pics[i].plane[p], name, p, who)) != 0) return rc;
        }
        if (g.planes == 2 && pics[i].plane[2])
            return fail(GLAVA_B200_EINVAL, "%s: pics[%d].plane[2] must be NULL: %s has one interleaved chroma plane", who, i,
                        planes_format_name(desc->format));
        if (g.planes == 1 && (pics[i].plane[1] || pics[i].plane[2]))
            return fail(GLAVA_B200_EINVAL, "%s: pics[%d].plane[%d] must be NULL: %s has one packed plane", who, i,
                        pics[i].plane[1] ? 1 : 2, planes_format_name(desc->format));
    }
    return 0;
}

// Two plane rectangles of pitches a.P, b.P and row bytes a.B, b.B, a starting first (a.p <= b.p).  Equal (P, B): rects_meet's
// exact divmod test.  Otherwise each row of b that starts before a's last row ends is tested against a's rows
// (rect_meets_range, exact); rows of b past that point start after every byte of a.
bool plane_rects_meet(const PlaneRect& a, const PlaneRect& b) {
    const Rect ra = { a.p, a.rows, a.entry, a.plane != 0 }, rb = { b.p, b.rows, b.entry, b.plane != 0 };
    if (a.P == b.P && a.B == b.B) return rects_meet(ra, rb, a.P, a.B);
    const uintptr_t end = a.p + (a.rows - 1) * a.P + a.B;
    for (size_t j = 0; j < b.rows && b.p + j * b.P < end; ++j)
        if (rect_meets_range(ra, a.P, a.B, b.p + j * b.P, b.p + j * b.P + b.B)) return true;
    return false;
}

int planes_geometry_check(int w, int h, int count, const glava_b200_picture* pics, const glava_b200_overlay_planes_desc& desc,
                          const uint8_t* const* fb, const size_t* fb_bytes, int nfb, const char* who, bool rgba) {
    PlanesGeom g;
    int rc = planes_geometry(w, h, desc, &g, who, rgba);
    if (rc) return rc;
    std::vector<PlaneRect> rs;
    rs.reserve((size_t) count * (size_t) g.planes);
    for (int i = 0; i < count; ++i)
        for (int p = 0; p < g.planes; ++p)
            rs.push_back(p == 0 ? PlaneRect{ (uintptr_t) pics[i].plane[0], (size_t) h, desc.pitch, g.luma_row, i, 0 }
                                : PlaneRect{ (uintptr_t) pics[i].plane[p], (size_t) g.chroma_rows, desc.chroma_pitch, g.chroma_row, i, p });
    for (const PlaneRect& r : rs) {
        const Rect q = { r.p, r.rows, r.entry, r.plane != 0 };
        for (int k = 0; k < nfb; ++k)
            if (rect_meets_range(q, r.P, r.B, (uintptr_t) fb[k], (uintptr_t) fb[k] + fb_bytes[k]))
                return fail(GLAVA_B200_EINVAL, "%s: the %s rectangle of entry %d overlaps the renderer's framebuffer", who,
                            plane_name(g.planes, r.plane), r.entry);
    }
    // by address: a rectangle can only meet those that start before its last row ends
    std::sort(rs.begin(), rs.end(), [](const PlaneRect& a, const PlaneRect& b) { return a.p < b.p; });
    for (size_t i = 0; i < rs.size(); ++i) {
        const uintptr_t end = rs[i].p + (rs[i].rows - 1) * rs[i].P + rs[i].B;
        for (size_t j = i + 1; j < rs.size() && rs[j].p < end; ++j)
            if (plane_rects_meet(rs[i], rs[j])) {
                const bool first = rs[i].entry < rs[j].entry || (rs[i].entry == rs[j].entry && rs[i].plane < rs[j].plane);
                const PlaneRect& a = first ? rs[i] : rs[j];
                const PlaneRect& b = first ? rs[j] : rs[i];
                return fail(GLAVA_B200_EINVAL, "%s: the %s rectangle of entry %d overlaps the %s rectangle of entry %d (layers go in "
                            "separate calls)", who, plane_name(g.planes, a.plane), a.entry,
                            plane_name(g.planes, b.plane), b.entry);
            }
    }
    return 0;
}

int planes_list(const RendererView& v, const int* streams, int count, const glava_b200_picture* pics, const uint8_t* k, int pad,
                ExportList** L, size_t* bytes) {
    int n = 0;
    for (int i = 0; i < count; ++i) n += !k || k[i] ? 1 : 0;
    *bytes = (size_t) n * sizeof(OverlayPlanesEntry);
    int rc;
    if ((rc = list_room(v, *bytes, L)) != 0) return rc;
    CU(cudaEventSynchronize((*L)->ev[(*L)->cur]));          // the copy that last read h[cur] (four calls ago)
    OverlayPlanesEntry* const host = reinterpret_cast<OverlayPlanesEntry*>((uint8_t*) (*L)->h[(*L)->cur]);
    for (int i = 0, j = 0; i < count; ++i)
        if (!k || k[i])
            host[j++] = { { (uint8_t*) pics[i].plane[0], (uint8_t*) pics[i].plane[1], (uint8_t*) pics[i].plane[2] }, streams[i] % v.slots,
                          k ? k[i] : pad };
    return 0;
}

// On the handle's stream, where readback copies: after the latest raster pass, before the next one can overwrite a slot
int planes_run(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics, const glava_b200_overlay_planes_desc* desc,
               void* after_event, void* done_event, const char* who, const uint8_t* opacity) {
    clear_error();
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = planes_check(r, streams, count, pics, desc, who);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    const size_t fb_bytes = (size_t) v.slots * (size_t) v.h * (size_t) v.w * 4;
    if ((rc = planes_geometry_check(v.w, v.h, count, pics, *desc, &v.fb, &fb_bytes, 1, who)) != 0) return rc;
    CU(cudaSetDevice(v.device));
    // opacity (DESIGN 4.20) as overlay_frames': the fade kernel unless every K is 255, K = 0 entries left out of the list
    const bool fade = opacity_fades(opacity, count);
    ExportList* L = nullptr;
    size_t bytes = 0;
    if ((rc = planes_list(v, streams, count, pics, fade ? opacity : nullptr, 0, &L, &bytes)) != 0) return rc;
    count = (int) (bytes / sizeof(OverlayPlanesEntry));
    return list_enqueue(v, L, bytes, after_event, done_event, [&](const void* d_list) {
        OverlayPlanesArgs a = {};
        a.fb = v.fb;
        a.marks = v.mark_key ? v.marks : nullptr;           // as export.cpp's common_args
        a.mark_rows = v.mark_key >> 2;
        a.list = static_cast<const OverlayPlanesEntry*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
        a.format = desc->format;
        a.native = v.native;
        a.band = a.native && a.marks && a.mark_rows > 0 ? 1 : 0;   // band items wherever marks exist, as overlay_frames
        a.pitch = desc->pitch; a.chroma_pitch = desc->chroma_pitch;
        a.enc = export_enc(desc->flags);
        a.fade = fade ? 1 : 0;
        return launch_overlay_planes(a, v.stream);
    });
}

}  // namespace glb

extern "C" int glava_b200_overlay_planes(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                                         const glava_b200_overlay_planes_desc* desc, void* after_event, void* done_event) {
    return glb::planes_run(r, streams, count, pics, desc, after_event, done_event, "glava_b200_overlay_planes");
}
extern "C" int glava_b200_overlay_planes_opacity(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                                                 const glava_b200_overlay_planes_desc* desc, const uint8_t* opacity,
                                                 void* after_event, void* done_event) {
    return glb::planes_run(r, streams, count, pics, desc, after_event, done_event, "glava_b200_overlay_planes_opacity", opacity);
}
