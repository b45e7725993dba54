// overlay.cpp — the host half of the overlay (DESIGN 4.12): glava_b200_overlay_frames and the checks
// glava_b200_sharded_overlay_frames runs before any shard starts.  The descriptor checks, destination checks and list
// buffers are export.cpp's; the kernel is export_kernels.cu overlay_kernel.
#include "internal.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace glb;

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

namespace {

// One plane of one entry's rectangle: `rows` rows of the common row bytes, the common pitch apart, from byte address p
struct Rect { uintptr_t p; size_t rows; int entry; bool uv; };

// Two rectangles of one pitch P and row bytes B, a starting first (a.p <= b.p): with q, m = divmod(b.p - a.p, P), b's row 0
// meets a's row q when m < B and a's row q + 1 when P - m < B, and b's later rows meet a's later rows only if row 0 does
bool rects_meet(const Rect& a, const Rect& b, size_t P, size_t B) {
    const uintptr_t d = b.p - a.p, q = d / P, m = d % P;
    return (q < a.rows && m < B) || (q + 1 < a.rows && P - m < B);
}

// whether rows of r meet the byte range [f0, f1)
bool rect_meets_range(const Rect& r, size_t P, size_t B, uintptr_t f0, uintptr_t f1) {
    if (f1 <= r.p || f0 >= r.p + (r.rows - 1) * P + B) return false;
    size_t k = f0 <= r.p ? 0 : (f0 - r.p) / P;              // the first row that ends past f0
    if (r.p + k * P + B <= f0) ++k;
    return k < r.rows && r.p + k * P < f1;
}

}  // namespace

namespace glb {
int overlay_check(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                  const glava_b200_export* desc, const char* who) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    int rc = export_desc_format(*desc, who);
    if (rc) return rc;
    if (desc->flags) return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: the overlay takes none", who, desc->flags);
    if ((rc = export_desc_size(v.w, v.h, *desc, "frame", who)) != 0) return rc;
    if (dst_uv && desc->format != GLAVA_B200_EXPORT_NV12) return fail(GLAVA_B200_EINVAL, "%s: dst_uv is for NV12 only", who);
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    for (int i = 0; i < count; ++i) {
        if (streams[i] < 0 || streams[i] >= v.batch)
            return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, streams[i], v.batch);
        if ((rc = export_dst_check(v, dst[i], "dst", i, who)) != 0) return rc;
        if (dst_uv && (rc = export_dst_check(v, dst_uv[i], "dst_uv", i, who)) != 0) return rc;
    }
    return 0;
}

int overlay_geometry_check(int w, int h, int count, void* const* dst, void* const* dst_uv, const glava_b200_export& desc,
                           const uint8_t* const* fb, const size_t* fb_bytes, int nfb, const char* who) {
    const bool nv12 = desc.format == GLAVA_B200_EXPORT_NV12;
    const size_t P = desc.pitch, B = nv12 ? (size_t) w : (size_t) w * 4;
    const size_t uv_offset = desc.uv_offset ? desc.uv_offset : P * (size_t) h;
    std::vector<Rect> rs;
    rs.reserve((size_t) count * (nv12 ? 2 : 1));
    for (int i = 0; i < count; ++i) {
        rs.push_back({ (uintptr_t) dst[i], (size_t) h, i, false });
        if (nv12) rs.push_back({ dst_uv ? (uintptr_t) dst_uv[i] : (uintptr_t) dst[i] + uv_offset, (size_t) h / 2, i, true });
    }
    for (const Rect& r : rs)
        for (int k = 0; k < nfb; ++k)
            if (rect_meets_range(r, P, B, (uintptr_t) fb[k], (uintptr_t) fb[k] + fb_bytes[k]))
                return fail(GLAVA_B200_EINVAL, "%s: the %s rectangle of entry %d overlaps the renderer's framebuffer", who,
                            r.uv ? "CbCr" : "destination", r.entry);
    // by address: a rectangle can only meet those that start before its last row ends
    std::sort(rs.begin(), rs.end(), [](const Rect& a, const Rect& b) { return a.p < b.p; });
    for (size_t i = 0; i < rs.size(); ++i) {
        const uintptr_t end = rs[i].p + (rs[i].rows - 1) * P + B;
        for (size_t j = i + 1; j < rs.size() && rs[j].p < end; ++j)
            if (rects_meet(rs[i], rs[j], P, B)) {
                const Rect& a = rs[i].entry < rs[j].entry ? rs[i] : rs[j];
                const Rect& b = rs[i].entry < rs[j].entry ? rs[j] : rs[i];
                return fail(GLAVA_B200_EINVAL, "%s: the %s rectangle of entry %d overlaps the %s rectangle of entry %d (layers go in "
                            "separate calls)", who, a.uv ? "CbCr" : "destination", a.entry, b.uv ? "CbCr" : "destination", b.entry);
            }
    }
    return 0;
}
}  // namespace glb

extern "C" {

// On the handle's stream, as glava_b200_export_frames
int glava_b200_overlay_frames(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                              const glava_b200_export* desc, void* after_event, void* done_event) {
    clear_error();
    const char* who = "glava_b200_overlay_frames";
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = overlay_check(r, streams, count, dst, dst_uv, desc, who);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    const size_t fb_bytes = (size_t) v.slots * (size_t) v.h * (size_t) v.w * 4;
    if ((rc = overlay_geometry_check(v.w, v.h, count, dst, dst_uv, *desc, &v.fb, &fb_bytes, 1, who)) != 0) return rc;
    const bool nv12 = desc->format == GLAVA_B200_EXPORT_NV12;
    const size_t uv_offset = desc->uv_offset ? desc->uv_offset : desc->pitch * (size_t) v.h;
    CU(cudaSetDevice(v.device));
    void* host = nullptr;
    const void* d_list = nullptr;
    const size_t bytes = (size_t) count * sizeof(OverlayEntry);
    if ((rc = export_list_begin(v, bytes, &host)) != 0) return rc;
    OverlayEntry* list = static_cast<OverlayEntry*>(host);
    for (int i = 0; i < count; ++i) {
        list[i].dst = (uint8_t*) dst[i];
        list[i].dst_uv = !nv12 ? nullptr : dst_uv ? (uint8_t*) dst_uv[i] : (uint8_t*) dst[i] + uv_offset;
        list[i].slot = streams[i] % v.slots; list[i].pad = 0;
    }
    if ((rc = export_list_end(v, bytes, after_event, &d_list)) != 0) return rc;
    OverlayArgs a = {};
    a.fb = v.fb;
    a.marks = v.mark_key ? v.marks : nullptr;              // as glava_b200_export_frames
    a.mark_rows = v.mark_key >> 2;
    a.list = static_cast<const OverlayEntry*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
    a.format = desc->format;
    a.native = v.native;
    // band items whenever they apply; GLAVA_B200_OVERLAY_ITEM=pair keeps row-pair items under marks (a measurement aid,
    // DESIGN 4.12)
    const char* item = getenv("GLAVA_B200_OVERLAY_ITEM");
    a.band = a.native && a.marks && a.mark_rows > 0 && !(item && !strcmp(item, "pair")) ? 1 : 0;
    a.pitch = desc->pitch;
    if ((rc = launch_overlay(a, v.stream)) != 0) return rc;
    ++*v.launches;
    if (done_event) CU(cudaEventRecord((cudaEvent_t) done_event, (cudaStream_t) v.stream));
    return 0;
}

}  // extern "C"
