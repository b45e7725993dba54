// export_list.h — what every caller-buffer export enqueues through (host code): the per-renderer list buffers kept in the
// renderer's attachment slot and the one enqueue sequence.  export.cpp (export_frames, export_scaled, overlay_frames)
// and export_ladder.cpp (export_ladder) share them.
#ifndef GLAVA_B200_EXPORT_LIST_H
#define GLAVA_B200_EXPORT_LIST_H

#include "internal.h"
#include "cuda_owner.h"

#include <cuda_runtime.h>

#include <vector>

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

namespace glb {

// The entry list of one renderer: it goes up from four pinned buffers in turn into one device list (read by the kernel on
// the raster stream, behind the copy that fills it), allocated on first use and grown to the longest list, in bytes so
// that either entry type (ExportEntry, ExportEntryUV) fits; ev[i]: the copy out of h[i] is done.  The ladder's schedule
// (ladder_plan.h) stays on the device for the geometry it was built for (sched_key), so a steady ladder uploads only its
// list; sched_h holds what went up until the copy has read it.
struct ExportList {
    PinnedBuf<uint8_t> h[4]; DevBuf<uint8_t> d; Event ev[4]; int cur = 0; size_t cap = 0;
    std::vector<int> sched_key; std::vector<uint64_t> sched_h; DevBuf<uint64_t> sched; size_t sched_cap = 0;
};

// room for `bytes` of list (the buffers are replaced only once the raster stream has drained); *out: the renderer's list
int list_room(const RendererView& v, size_t bytes, ExportList** out);

// overlay_planes.cpp: the list of an overlay onto pictures (overlay_planes, DESIGN 4.17; overlay_scaled, 4.21) in the pinned
// buffer h[cur] of the renderer's list: one OverlayPlanesEntry (plane pointers, slot) per entry whose K is not 0, K in its pad
// word; k null: every entry, pad `pad`.  *bytes: the list's size.
int planes_list(const RendererView& v, const int* streams, int count, const glava_b200_picture* pics, const uint8_t* k, int pad,
                ExportList** L, size_t* bytes);

// the background of a descriptor as 0x00BBGGRR
uint32_t background(const glava_b200_export& d);

// (export.cpp, shared with overlay_planes.cpp) a destination pointer: null, 16-byte alignment, device memory, the
// renderer's device; `name`[i] names it in the message
int dst_check(const RendererView& v, const void* p, const char* name, int i, const char* who);
// the HDR bits of a descriptor that has one (export.cpp, DESIGN 4.22)
int hdr_flags_check(int format, uint32_t flags, const char* who);
// One plane of one entry's rectangle: `rows` rows of the common row bytes, the common pitch apart, from byte address p
struct Rect { uintptr_t p; size_t rows; int entry; bool uv; };
// Two rectangles of one pitch P and row bytes B, a starting first (a.p <= b.p): whether any rows meet
bool rects_meet(const Rect& a, const Rect& b, size_t P, size_t B);
// whether rows of r meet the byte range [f0, f1)
bool rect_meets_range(const Rect& r, size_t P, size_t B, uintptr_t f0, uintptr_t f1);

// whether an overlay's opacity list ([count] K, null: all 255) needs the fade kernels (DESIGN 4.20): some K is not 255
inline bool opacity_fades(const uint8_t* opacity, int count) {
    for (int i = 0; opacity && i < count; ++i)
        if (opacity[i] != 255) return true;
    return false;
}

// The enqueue every call shares, on the raster stream: wait for after_event, copy the list out of the pinned buffer the
// caller filled (h[cur]) and record its event, launch(device list), then done_event.  An empty list (an overlay whose every
// entry is at opacity 0) copies and launches nothing: the stream still waits for after_event and records done_event.
template <typename Launch>
int list_enqueue(const RendererView& v, ExportList* L, size_t bytes, void* after_event, void* done_event, Launch launch) {
    cudaStream_t st = (cudaStream_t) v.stream;
    const int k = L->cur;
    if (after_event) CU(cudaStreamWaitEvent(st, (cudaEvent_t) after_event, 0));
    if (!bytes) {
        if (done_event) CU(cudaEventRecord((cudaEvent_t) done_event, st));
        return 0;
    }
    CU(cudaMemcpyAsync(L->d, L->h[k], bytes, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(L->ev[k], st));
    L->cur = (k + 1) & 3;
    const int rc = launch((const void*) L->d);
    if (rc) return rc;
    ++*v.launches;
    if (done_event) CU(cudaEventRecord((cudaEvent_t) done_event, st));
    return 0;
}

}  // namespace glb
#endif
