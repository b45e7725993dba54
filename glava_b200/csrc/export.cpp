// export.cpp — the host half of frame export (DESIGN 4.10): glava_b200_export_bytes, glava_b200_export_frames and the
// checks glava_b200_sharded_export_frames runs before any shard starts.  It reads the renderer through capi.cu's
// renderer_view and keeps its list buffers in the renderer's attachment slot; the kernel is export_kernels.cu.
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
// kernel on the raster stream, behind the copy that fills it), allocated on first use and grown to the longest list;
// ev[i]: the copy out of h[i] is done
struct ExportList {
    PinnedBuf<ExportEntry> h[4]; DevBuf<ExportEntry> d; Event ev[4]; int cur = 0, cap = 0;
};
void release_list(void* p) { delete static_cast<ExportList*>(p); }

// The checks of a descriptor against a w x h frame (glava_b200_export_bytes and every export)
int desc_check(int w, int h, const glava_b200_export& d, const char* who) {
    const bool nv12 = d.format == GLAVA_B200_EXPORT_NV12;
    if (d.format != GLAVA_B200_EXPORT_RGBA && d.format != GLAVA_B200_EXPORT_BGRA && !nv12)
        return fail(GLAVA_B200_EINVAL, "%s: unknown format %d", who, d.format);
    if (d.flags & ~GLAVA_B200_EXPORT_OVER) return fail(GLAVA_B200_EINVAL, "%s: unknown flags 0x%x", who, d.flags);
    if (nv12 && ((w | h) & 1)) return fail(GLAVA_B200_EINVAL, "%s: NV12 needs an even width and height, the frame is %dx%d", who, w, h);
    const size_t row = nv12 ? (size_t) w : (size_t) w * 4;
    if (d.pitch % 16 || d.pitch < row)
        return fail(GLAVA_B200_EINVAL, "%s: pitch %zu must be a multiple of 16 and at least %zu", who, d.pitch, row);
    if (nv12 && (d.uv_offset % 16 || (d.uv_offset && d.uv_offset < d.pitch * (size_t) h)))
        return fail(GLAVA_B200_EINVAL, "%s: uv_offset %zu must be a multiple of 16 and at least pitch * h = %zu (or 0)", who,
                    d.uv_offset, d.pitch * (size_t) h);
    return 0;
}

// room for `count` entries (the buffers are replaced only once the raster stream has drained)
int list_room(const RendererView& v, int count, ExportList** out) {
    if (!*v.attach) {
        *v.attach = new ExportList();
        *v.attach_free = release_list;
    }
    ExportList* L = static_cast<ExportList*>(*v.attach);
    *out = L;
    int rc;
    if (!L->ev[3].get())                                    // created last: the four events are complete
        for (Event& e : L->ev) if ((rc = e.create()) != 0) return rc;
    if (count <= L->cap) return 0;
    CU(cudaStreamSynchronize((cudaStream_t) v.stream));
    L->cap = 0;
    int cap = 64;
    while (cap < count) cap *= 2;
    const size_t bytes = (size_t) cap * sizeof(ExportEntry);
    if ((rc = L->d.alloc(bytes)) != 0) return rc;
    for (PinnedBuf<ExportEntry>& h : L->h) if ((rc = h.alloc(bytes)) != 0) return rc;
    L->cap = cap;
    return 0;
}

}  // namespace

namespace glb {
int export_check(glava_b200* r, const int* streams, int count, void* const* dst, const glava_b200_export* desc, const char* who) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    int rc = desc_check(v.w, v.h, *desc, who);
    if (rc) return rc;
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    for (int i = 0; i < count; ++i) {
        if (streams[i] < 0 || streams[i] >= v.batch)
            return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, streams[i], v.batch);
        if (!dst[i] || ((uintptr_t) dst[i] & 15))
            return fail(GLAVA_B200_EINVAL, "%s: dst[%d] = %p is null or not 16-byte aligned", who, i, dst[i]);
        cudaPointerAttributes at;
        memset(&at, 0, sizeof(at));
        if (cudaPointerGetAttributes(&at, dst[i]) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
        if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged)
            return fail(GLAVA_B200_EINVAL, "%s: dst[%d] = %p is not device memory", who, i, dst[i]);
        if (at.device != v.device)
            return fail(GLAVA_B200_EINVAL, "%s: dst[%d] is on device %d, the renderer on device %d", who, i, at.device, v.device);
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
    int rc = desc_check(p.w, p.h, *desc, who);
    if (rc) return rc;
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
    ExportList* L = nullptr;
    if ((rc = list_room(v, count, &L)) != 0) return rc;
    const int k = L->cur;
    CU(cudaEventSynchronize(L->ev[k]));                     // the copy that last read h[k] (four exports ago)
    ExportEntry* list = L->h[k];
    for (int i = 0; i < count; ++i) {
        list[i].dst = (uint8_t*) dst[i]; list[i].slot = streams[i] % v.slots; list[i].pad = 0;
    }
    if (after_event) CU(cudaStreamWaitEvent(st, (cudaEvent_t) after_event, 0));
    CU(cudaMemcpyAsync(L->d, list, (size_t) count * sizeof(ExportEntry), cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(L->ev[k], st));
    L->cur = (k + 1) & 3;
    ExportArgs a = {};
    a.fb = v.fb;
    // marks the last raster pass kept describe the framebuffer, whatever GLAVA_B200_FULL_STORE says (it only makes that pass
    // store every zero row); mark_key 0: none, or a kernel that keeps none wrote the frame since
    a.marks = v.mark_key ? v.marks : nullptr;
    a.mark_rows = v.mark_key >> 2;
    a.list = L->d; a.count = count; a.w = v.w; a.h = v.h;
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
