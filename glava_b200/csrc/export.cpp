// export.cpp — the host half of frame export (DESIGN 4.10): glava_b200_export_bytes, glava_b200_export_frames and the
// checks glava_b200_sharded_export_frames runs before any shard starts.  It reads the renderer through capi.cu's
// renderer_view and keeps its list buffers in the renderer's attachment slot; the kernel is export_kernels.cu.  The
// descriptor and destination checks and the list buffers also serve the scaled export (export_scaled.cpp).
#include "internal.h"
#include "cuda_owner.h"

#include <cuda_runtime.h>

#include <cstring>

using namespace glb;

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

namespace {

// The entry list of one renderer: it goes up from four pinned buffers in turn into one device list (read by the export
// kernel on the raster stream, behind the copy that fills it), allocated on first use and grown to the longest list, in
// bytes so that either entry type (ExportEntry, ScaledEntry) fits; ev[i]: the copy out of h[i] is done
struct ExportList {
    PinnedBuf<uint8_t> h[4]; DevBuf<uint8_t> d; Event ev[4]; int cur = 0; size_t cap = 0;
};
void release_list(void* p) { delete static_cast<ExportList*>(p); }

// room for `bytes` of list (the buffers are replaced only once the raster stream has drained)
int list_room(const RendererView& v, size_t bytes, ExportList** out) {
    if (!*v.attach) {
        *v.attach = new ExportList();
        *v.attach_free = release_list;
    }
    ExportList* L = static_cast<ExportList*>(*v.attach);
    *out = L;
    int rc;
    if (!L->ev[3].get())                                    // created last: the four events are complete
        for (Event& e : L->ev) if ((rc = e.create()) != 0) return rc;
    if (bytes <= L->cap) return 0;
    CU(cudaStreamSynchronize((cudaStream_t) v.stream));
    L->cap = 0;
    size_t cap = 64 * sizeof(ExportEntry);
    while (cap < bytes) cap *= 2;
    if ((rc = L->d.alloc(cap)) != 0) return rc;
    for (PinnedBuf<uint8_t>& h : L->h) if ((rc = h.alloc(cap)) != 0) return rc;
    L->cap = cap;
    return 0;
}

}  // namespace

namespace glb {
// The checks of a descriptor: format and flags, then pitch and uv_offset against a w x h output
int export_desc_format(const glava_b200_export& d, const char* who) {
    if (d.format != GLAVA_B200_EXPORT_RGBA && d.format != GLAVA_B200_EXPORT_BGRA && d.format != GLAVA_B200_EXPORT_NV12)
        return fail(GLAVA_B200_EINVAL, "%s: unknown format %d", who, d.format);
    if (d.flags & ~GLAVA_B200_EXPORT_OVER) return fail(GLAVA_B200_EINVAL, "%s: unknown flags 0x%x", who, d.flags);
    return 0;
}
int export_desc_size(int w, int h, const glava_b200_export& d, const char* what, const char* who) {
    const bool nv12 = d.format == GLAVA_B200_EXPORT_NV12;
    if (nv12 && ((w | h) & 1)) return fail(GLAVA_B200_EINVAL, "%s: NV12 needs an even width and height, the %s is %dx%d", who, what, w, h);
    const size_t row = nv12 ? (size_t) w : (size_t) w * 4;
    if (d.pitch % 16 || d.pitch < row)
        return fail(GLAVA_B200_EINVAL, "%s: pitch %zu must be a multiple of 16 and at least %zu", who, d.pitch, row);
    if (nv12 && (d.uv_offset % 16 || (d.uv_offset && d.uv_offset < d.pitch * (size_t) h)))
        return fail(GLAVA_B200_EINVAL, "%s: uv_offset %zu must be a multiple of 16 and at least pitch * h = %zu (or 0)", who,
                    d.uv_offset, d.pitch * (size_t) h);
    return 0;
}

int export_dst_check(const RendererView& v, const void* p, const char* name, int i, const char* who) {
    if (!p || ((uintptr_t) p & 15))
        return fail(GLAVA_B200_EINVAL, "%s: %s[%d] = %p is null or not 16-byte aligned", who, name, i, p);
    cudaPointerAttributes at;
    memset(&at, 0, sizeof(at));
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged)
        return fail(GLAVA_B200_EINVAL, "%s: %s[%d] = %p is not device memory", who, name, i, p);
    if (at.device != v.device)
        return fail(GLAVA_B200_EINVAL, "%s: %s[%d] is on device %d, the renderer on device %d", who, name, i, at.device, v.device);
    return 0;
}

int export_list_begin(const RendererView& v, size_t bytes, void** host) {
    ExportList* L = nullptr;
    int rc;
    if ((rc = list_room(v, bytes, &L)) != 0) return rc;
    CU(cudaEventSynchronize(L->ev[L->cur]));                // the copy that last read h[cur] (four exports ago)
    *host = L->h[L->cur];
    return 0;
}

int export_list_end(const RendererView& v, size_t bytes, void* after_event, const void** d_list) {
    ExportList* L = static_cast<ExportList*>(*v.attach);
    cudaStream_t st = (cudaStream_t) v.stream;
    const int k = L->cur;
    if (after_event) CU(cudaStreamWaitEvent(st, (cudaEvent_t) after_event, 0));
    CU(cudaMemcpyAsync(L->d, L->h[k], bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(L->ev[k], st));
    L->cur = (k + 1) & 3;
    *d_list = L->d;
    return 0;
}

int export_check(glava_b200* r, const int* streams, int count, void* const* dst, const glava_b200_export* desc, const char* who) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    int rc = export_desc_format(*desc, who);
    if (rc || (rc = export_desc_size(v.w, v.h, *desc, "frame", who)) != 0) return rc;
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    for (int i = 0; i < count; ++i) {
        if (streams[i] < 0 || streams[i] >= v.batch)
            return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, streams[i], v.batch);
        if ((rc = export_dst_check(v, dst[i], "dst", i, who)) != 0) return rc;
    }
    return 0;
}
}  // namespace glb

extern "C" {

int glava_b200_export_bytes(const glava_b200* r, const glava_b200_export* desc, size_t* bytes) {
    clear_error();
    const char* who = "glava_b200_export_bytes";
    glava_b200_params p;
    if (!r || !desc || !bytes || glava_b200_get_params(r, &p) != 0) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = export_desc_format(*desc, who);
    if (rc || (rc = export_desc_size(p.w, p.h, *desc, "frame", who)) != 0) return rc;
    const size_t h = (size_t) p.h;
    if (desc->format != GLAVA_B200_EXPORT_NV12) *bytes = desc->pitch * h;
    else *bytes = (desc->uv_offset ? desc->uv_offset : desc->pitch * h) + desc->pitch * (h / 2);
    return 0;
}

// On the handle's stream, where readback copies: after the latest raster pass, before the next one can overwrite a slot
int glava_b200_export_frames(glava_b200* r, const int* streams, int count, void* const* dst, const glava_b200_export* desc,
                             void* after_event, void* done_event) {
    clear_error();
    const char* who = "glava_b200_export_frames";
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = export_check(r, streams, count, dst, desc, who);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    cudaStream_t st = (cudaStream_t) v.stream;
    CU(cudaSetDevice(v.device));
    void* host = nullptr;
    const void* d_list = nullptr;
    if ((rc = export_list_begin(v, (size_t) count * sizeof(ExportEntry), &host)) != 0) return rc;
    ExportEntry* list = static_cast<ExportEntry*>(host);
    for (int i = 0; i < count; ++i) {
        list[i].dst = (uint8_t*) dst[i]; list[i].slot = streams[i] % v.slots; list[i].pad = 0;
    }
    if ((rc = export_list_end(v, (size_t) count * sizeof(ExportEntry), after_event, &d_list)) != 0) return rc;
    ExportArgs a = {};
    a.fb = v.fb;
    // marks the last raster pass kept describe the framebuffer, whatever GLAVA_B200_FULL_STORE says (it only makes that pass
    // store every zero row); mark_key 0: none, or a kernel that keeps none wrote the frame since
    a.marks = v.mark_key ? v.marks : nullptr;
    a.mark_rows = v.mark_key >> 2;
    a.list = static_cast<const ExportEntry*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
    a.format = desc->format;
    a.over = desc->format == GLAVA_B200_EXPORT_NV12 || (desc->flags & GLAVA_B200_EXPORT_OVER) ? 1 : 0;
    a.native = v.native;
    a.bg = (uint32_t) desc->background[0] | ((uint32_t) desc->background[1] << 8) | ((uint32_t) desc->background[2] << 16);
    a.pitch = desc->pitch;
    a.uv_offset = desc->uv_offset ? desc->uv_offset : desc->pitch * (size_t) v.h;
    if ((rc = launch_export(a, st)) != 0) return rc;
    ++*v.launches;
    if (done_event) CU(cudaEventRecord((cudaEvent_t) done_event, st));
    return 0;
}

}  // extern "C"
