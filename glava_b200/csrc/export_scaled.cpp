// export_scaled.cpp — the host half of the scaled and cropped export (DESIGN 4.11): glava_b200_export_scaled_bytes,
// glava_b200_export_scaled and the checks glava_b200_sharded_export_scaled runs before any shard starts.  The descriptor
// checks, destination checks and list buffers are export.cpp's; the kernel is export_kernels.cu export_scaled_kernel.
#include "internal.h"
#include "export_core.h"

#include <cuda_runtime.h>

using namespace glb;

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

namespace {

// The descriptor and the rectangle against a w x h frame: *q is the rectangle with the whole-frame default applied
int scale_check(int w, int h, const glava_b200_export& d, const glava_b200_export_scale* s, glava_b200_export_scale* q,
                const char* who) {
    int rc = export_desc_format(d, who);
    if (rc) return rc;
    if (!s) return fail(GLAVA_B200_EINVAL, "%s: null scale", who);
    *q = *s;
    if (!q->src_x && !q->src_y && !q->src_w && !q->src_h) { q->src_w = w; q->src_h = h; }
    if (q->src_x < 0 || q->src_y < 0 || q->src_w < 1 || q->src_h < 1 || (int64_t) q->src_x + q->src_w > w ||
        (int64_t) q->src_y + q->src_h > h)
        return fail(GLAVA_B200_EINVAL, "%s: source rectangle (%d, %d) %dx%d is empty or leaves the %dx%d frame", who, q->src_x,
                    q->src_y, q->src_w, q->src_h, w, h);
    if (q->out_w < 1 || q->out_h < 1 || q->out_w > q->src_w || q->out_h > q->src_h)
        return fail(GLAVA_B200_EINVAL, "%s: output %dx%d must be at least 1x1 and at most the %dx%d source (no upscaling)", who,
                    q->out_w, q->out_h, q->src_w, q->src_h);
    return export_desc_size(q->out_w, q->out_h, d, "output", who);
}

}  // namespace

namespace glb {
int export_scaled_check(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                        const glava_b200_export* desc, const glava_b200_export_scale* scale, const char* who) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    glava_b200_export_scale q;
    int rc = scale_check(v.w, v.h, *desc, scale, &q, who);
    if (rc) return rc;
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
}  // namespace glb

extern "C" {

int glava_b200_export_scaled_bytes(const glava_b200* r, const glava_b200_export* desc, const glava_b200_export_scale* scale,
                                   size_t* bytes) {
    clear_error();
    const char* who = "glava_b200_export_scaled_bytes";
    glava_b200_params p;
    if (!r || !desc || !bytes || glava_b200_get_params(r, &p) != 0) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_export_scale q;
    int rc = scale_check(p.w, p.h, *desc, scale, &q, who);
    if (rc) return rc;
    const size_t h = (size_t) q.out_h;
    if (desc->format != GLAVA_B200_EXPORT_NV12) *bytes = desc->pitch * h;
    else *bytes = (desc->uv_offset ? desc->uv_offset : desc->pitch * h) + desc->pitch * (h / 2);
    return 0;
}

// On the handle's stream, as glava_b200_export_frames
int glava_b200_export_scaled(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                             const glava_b200_export* desc, const glava_b200_export_scale* scale, void* after_event,
                             void* done_event) {
    clear_error();
    const char* who = "glava_b200_export_scaled";
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = export_scaled_check(r, streams, count, dst, dst_uv, desc, scale, who);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    glava_b200_export_scale q;
    scale_check(v.w, v.h, *desc, scale, &q, who);
    const bool nv12 = desc->format == GLAVA_B200_EXPORT_NV12;
    const size_t uv_offset = desc->uv_offset ? desc->uv_offset : desc->pitch * (size_t) q.out_h;
    CU(cudaSetDevice(v.device));
    void* host = nullptr;
    const void* d_list = nullptr;
    const size_t bytes = (size_t) count * sizeof(ScaledEntry);
    if ((rc = export_list_begin(v, bytes, &host)) != 0) return rc;
    ScaledEntry* list = static_cast<ScaledEntry*>(host);
    for (int i = 0; i < count; ++i) {
        list[i].dst = (uint8_t*) dst[i];
        list[i].dst_uv = !nv12 ? nullptr : dst_uv ? (uint8_t*) dst_uv[i] : (uint8_t*) dst[i] + uv_offset;
        list[i].slot = streams[i] % v.slots; list[i].pad = 0;
    }
    if ((rc = export_list_end(v, bytes, after_event, &d_list)) != 0) return rc;
    ScaledArgs a = {};
    a.fb = v.fb;
    a.marks = v.mark_key ? v.marks : nullptr;              // as glava_b200_export_frames
    a.mark_rows = v.mark_key >> 2;
    a.list = static_cast<const ScaledEntry*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
    a.format = desc->format;
    a.over = nv12 || (desc->flags & GLAVA_B200_EXPORT_OVER) ? 1 : 0;
    a.native = v.native;
    a.bg = (uint32_t) desc->background[0] | ((uint32_t) desc->background[1] << 8) | ((uint32_t) desc->background[2] << 16);
    a.pitch = desc->pitch;
    a.src_x = q.src_x; a.src_y = q.src_y; a.src_w = q.src_w; a.src_h = q.src_h; a.out_w = q.out_w; a.out_h = q.out_h;
    const ExportRecip rcp = export_recip((uint64_t) q.src_w * (uint64_t) q.src_h);
    a.div_mul = rcp.mul; a.div_shift = rcp.shift;
    if ((rc = launch_export_scaled(a, v.stream)) != 0) return rc;
    ++*v.launches;
    if (done_event) CU(cudaEventRecord((cudaEvent_t) done_event, (cudaStream_t) v.stream));
    return 0;
}

}  // extern "C"
