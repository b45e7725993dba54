// export.cpp — the host half of the three caller-buffer exports (DESIGN 4.10–4.12): glava_b200_export_frames,
// glava_b200_export_scaled and glava_b200_overlay_frames, their byte counts, and the checks the sharded forms run before any
// shard starts.  The three calls share one check, one list fill and one enqueue; what differs by kind is the output size
// (the frame, or the scale rectangle's), the flags allowed, and the kernel's own argument fields.  It reads the renderer
// through capi.cu's renderer_view and keeps its list buffers in the renderer's attachment slot; the kernels are
// export_kernels.cu.  The list buffers and the enqueue are export_list.h's, shared with the ladder (export_ladder.cpp).
#include "internal.h"
#include "export_core.h"
#include "export_list.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

using namespace glb;

namespace {

const char* const kCallName[] = { "glava_b200_export_frames", "glava_b200_export_scaled", "glava_b200_overlay_frames" };

const char* format_name(int format) {
    switch (format) {
    case GLAVA_B200_EXPORT_RGBA: return "RGBA";
    case GLAVA_B200_EXPORT_BGRA: return "BGRA";
    case GLAVA_B200_EXPORT_NV12: return "NV12";
    case GLAVA_B200_EXPORT_I420: return "I420";
    case GLAVA_B200_EXPORT_YUV444: return "YUV444";
    case GLAVA_B200_EXPORT_P010: return "P010";
    case GLAVA_B200_EXPORT_YUV420P10: return "YUV420P10";
    case GLAVA_B200_EXPORT_YUV444P10: return "YUV444P10";
    case GLAVA_B200_EXPORT_YUV422P: return "YUV422P";
    case GLAVA_B200_EXPORT_YUV422P10: return "YUV422P10";
    case GLAVA_B200_EXPORT_UYVY: return "UYVY";
    case GLAVA_B200_EXPORT_YUVA420P: return "YUVA420P";
    case GLAVA_B200_EXPORT_YUVA444P10: return "YUVA444P10";
    default: return nullptr;
    }
}

// pitch and uv_offset against a w x h output (`what` names it in the message: "frame" / "output")
int desc_size(int w, int h, const glava_b200_export& d, const char* what, const char* who) {
    const int fmt = d.format;
    const char* name = format_name(fmt);
    if (export_420(fmt) && ((w | h) & 1))
        return fail(GLAVA_B200_EINVAL, "%s: %s needs an even width and height, the %s is %dx%d", who, name, what, w, h);
    if (export_422(fmt) && (w & 1))                         // chroma per pixel pair; 4:2:2 rows are independent, any h
        return fail(GLAVA_B200_EINVAL, "%s: %s needs an even width, the %s is %dx%d", who, name, what, w, h);
    const size_t row = !export_ycbcr(fmt) ? (size_t) w * 4
                       : fmt == GLAVA_B200_EXPORT_P010 || export_p10(fmt) || fmt == GLAVA_B200_EXPORT_YUV422P10 ||
                                 fmt == GLAVA_B200_EXPORT_UYVY || fmt == GLAVA_B200_EXPORT_YUVA444P10
                           ? (size_t) w * 2
                           : (size_t) w;
    if (d.pitch % 16 || d.pitch < row)
        return fail(GLAVA_B200_EINVAL, "%s: pitch %zu must be a multiple of 16 and at least %zu", who, d.pitch, row);
    if ((fmt == GLAVA_B200_EXPORT_I420 || fmt == GLAVA_B200_EXPORT_YUV420P10 || fmt == GLAVA_B200_EXPORT_YUV422P ||
         fmt == GLAVA_B200_EXPORT_YUV422P10 || fmt == GLAVA_B200_EXPORT_YUVA420P) && d.pitch % 32)
        return fail(GLAVA_B200_EINVAL, "%s: %s pitch %zu must be a multiple of 32, so that chroma rows (pitch / 2) stay 16-byte "
                    "aligned", who, name, d.pitch);
    if ((fmt == GLAVA_B200_EXPORT_NV12 || fmt == GLAVA_B200_EXPORT_P010) &&
        (d.uv_offset % 16 || (d.uv_offset && d.uv_offset < d.pitch * (size_t) h)))
        return fail(GLAVA_B200_EINVAL, "%s: uv_offset %zu must be a multiple of 16 and at least pitch * h = %zu (or 0)", who,
                    d.uv_offset, d.pitch * (size_t) h);
    if (fmt == GLAVA_B200_EXPORT_UYVY && d.uv_offset)
        return fail(GLAVA_B200_EINVAL, "%s: UYVY uv_offset %zu must be 0: UYVY has no chroma plane", who, d.uv_offset);
    const size_t plane = export_planes(fmt, d.pitch, 0, h).plane;
    if (export_planar(fmt) && (d.uv_offset % 16 || (d.uv_offset && d.uv_offset < plane)))
        return fail(GLAVA_B200_EINVAL, "%s: %s uv_offset %zu (Cb plane to Cr plane) must be a multiple of 16 and at least one "
                    "chroma plane, %zu bytes (or 0)", who, name, d.uv_offset, plane);
    return 0;
}

// The descriptor of a call of `kind` against a w x h frame: format and flags, the scale rectangle (the scaled export
// only), then pitch and uv_offset against the output.  *q: the rectangle with the whole-frame default applied (the
// whole frame at its own size for the other kinds), so q->out_w x q->out_h is the output size.
int desc_check(ExportKind kind, int w, int h, const glava_b200_export& d, const glava_b200_export_scale* s,
               glava_b200_export_scale* q, const char* who) {
    if (!format_name(d.format)) return fail(GLAVA_B200_EINVAL, "%s: unknown format %d", who, d.format);
    if (kind == ExportKind::overlay && d.format != GLAVA_B200_EXPORT_NV12 && export_ycbcr(d.format))
        return fail(GLAVA_B200_EINVAL, "%s: format %s: the overlay takes RGBA, BGRA or NV12", who, format_name(d.format));
    // the colour bits (DESIGN 4.15) are flags of the Y'CbCr formats only
    const uint32_t colour = GLAVA_B200_EXPORT_FULL_RANGE | GLAVA_B200_EXPORT_BT601;
    const uint32_t hdr = GLAVA_B200_EXPORT_PQ | GLAVA_B200_EXPORT_HLG;
    if (d.flags & ~(GLAVA_B200_EXPORT_OVER | GLAVA_B200_EXPORT_STRAIGHT | colour | hdr))
        return fail(GLAVA_B200_EINVAL, "%s: unknown flags 0x%x", who, d.flags);
    if (d.flags & hdr) {                                    // DESIGN 4.22
        if (kind == ExportKind::overlay)
            return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: the overlay of RGBA, BGRA and NV12 takes no HDR bit (EXPORT_PQ, "
                        "EXPORT_HLG); HDR pictures go to glava_b200_overlay_planes", who, d.flags);
        const int rc = hdr_flags_check(d.format, d.flags, who);
        if (rc) return rc;
    }
    // transparency (DESIGN 4.19): straight alpha is RGBA / BGRA's alone, and never composited; the YUVA formats never are
    if (kind == ExportKind::overlay && (d.flags & GLAVA_B200_EXPORT_STRAIGHT))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_STRAIGHT is for the exports; the overlay composites", who, d.flags);
    if ((d.flags & GLAVA_B200_EXPORT_STRAIGHT) && (d.flags & GLAVA_B200_EXPORT_OVER))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_STRAIGHT and EXPORT_OVER exclude each other (a composite is "
                    "opaque)", who, d.flags);
    if ((d.flags & GLAVA_B200_EXPORT_STRAIGHT) && export_ycbcr(d.format))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_STRAIGHT is for RGBA and BGRA, not %s (YUVA420P and YUVA444P10 carry "
                    "straight alpha)", who, d.flags, format_name(d.format));
    if ((d.flags & GLAVA_B200_EXPORT_OVER) && export_yuva(d.format))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: %s is never composited (EXPORT_OVER), its A plane holds the frame's "
                    "alpha", who, d.flags, format_name(d.format));
    if ((d.flags & colour) && !export_ycbcr(d.format))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: %s has no matrix or range (EXPORT_FULL_RANGE and EXPORT_BT601 are for the "
                    "Y'CbCr formats)", who, d.flags, format_name(d.format));
    if (kind == ExportKind::overlay && (d.flags & ~colour))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: the overlay takes none%s", who, d.flags,
                    export_ycbcr(d.format) ? " but EXPORT_FULL_RANGE and EXPORT_BT601" : "");
    *q = { 0, 0, w, h, w, h };
    if (kind != ExportKind::scaled) return desc_size(w, h, d, "frame", who);
    const int rc = scale_check(w, h, s, q, who);
    return rc ? rc : desc_size(q->out_w, q->out_h, d, "output", who);
}

// the byte count of one destination of a call of `kind`
int output_bytes(ExportKind kind, const glava_b200* r, const glava_b200_export* desc, const glava_b200_export_scale* scale,
                 size_t* bytes, const char* who) {
    clear_error();
    glava_b200_params p;
    if (!r || !desc || !bytes || glava_b200_get_params(r, &p) != 0) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_export_scale q;
    const int rc = desc_check(kind, p.w, p.h, *desc, scale, &q, who);
    if (rc) return rc;
    const size_t h = (size_t) q.out_h;
    const ExportPlanes pl = export_planes(desc->format, desc->pitch, desc->uv_offset, q.out_h);
    if (!export_chroma_planes(desc->format)) *bytes = desc->pitch * h;   // RGBA, BGRA, UYVY: one plane
    else if (export_yuva(desc->format)) *bytes = pl.cb + 2 * pl.cr + desc->pitch * h;   // A: pitch * h, past Cr
    else if (export_planar(desc->format)) *bytes = pl.cb + pl.cr + pl.plane;
    else *bytes = pl.cb + desc->pitch * (h / 2);
    return 0;
}

// The fields every kind's argument struct has (they share names and meaning)
template <typename Args>
void common_args(Args& a, const RendererView& v, const void* d_list, int count, const glava_b200_export& d) {
    a.fb = v.fb;
    // marks the last raster pass kept describe the framebuffer, whatever GLAVA_B200_FULL_STORE says (it only makes that pass
    // store every zero row); mark_key 0: none, or a kernel that keeps none wrote the frame since
    a.marks = v.mark_key ? v.marks : nullptr;
    a.mark_rows = v.mark_key >> 2;
    a.list = static_cast<decltype(a.list)>(d_list); a.count = count; a.w = v.w; a.h = v.h;
    a.format = export_kernel_format(d.format, d.flags);
    a.native = v.native;
    a.pitch = d.pitch;
}

}  // namespace

namespace glb {
// The HDR bits (DESIGN 4.22) of an export or a picture: one of them, alone among the colour bits, without EXPORT_STRAIGHT,
// on P010, YUV420P10, YUV444P10 or YUV422P10
int hdr_flags_check(int format, uint32_t flags, const char* who) {
    const uint32_t hdr = GLAVA_B200_EXPORT_PQ | GLAVA_B200_EXPORT_HLG;
    if ((flags & hdr) == hdr)
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_PQ and EXPORT_HLG exclude each other", who, flags);
    if (flags & (GLAVA_B200_EXPORT_FULL_RANGE | GLAVA_B200_EXPORT_BT601))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_PQ / EXPORT_HLG are BT.2020 limited range (no EXPORT_FULL_RANGE or "
                    "EXPORT_BT601)", who, flags);
    if (flags & GLAVA_B200_EXPORT_STRAIGHT)
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_PQ / EXPORT_HLG carry no alpha (no EXPORT_STRAIGHT)", who, flags);
    if (!export_hdr_format(format))
        return fail(GLAVA_B200_EINVAL, "%s: flags 0x%x: EXPORT_PQ / EXPORT_HLG are for P010, YUV420P10, YUV444P10 and YUV422P10, "
                    "not format %d", who, flags, format);
    return 0;
}

int scale_check(int w, int h, const glava_b200_export_scale* s, glava_b200_export_scale* q, const char* who) {
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
    return 0;
}

// a destination pointer: null, alignment, device memory, device (export_list.h)
int dst_check(const RendererView& v, const void* p, const char* name, int i, const char* who) {
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

static void release_list(void* p) { delete static_cast<ExportList*>(p); }

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

uint32_t background(const glava_b200_export& d) {
    return (uint32_t) d.background[0] | ((uint32_t) d.background[1] << 8) | ((uint32_t) d.background[2] << 16);
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

int export_check(ExportKind kind, glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                 const glava_b200_export* desc, const glava_b200_export_scale* scale, const char* who, glava_b200_export_scale* q) {
    const RendererView v = renderer_view(r);
    if (!v.built) return fail(GLAVA_B200_EINVAL, "%s: the renderer has no tables: a reconfigure or resize failed and must be repeated", who);
    glava_b200_export_scale local;
    int rc = desc_check(kind, v.w, v.h, *desc, scale, q ? q : &local, who);
    if (rc) return rc;
    if (dst_uv && !export_chroma_planes(desc->format))
        return fail(GLAVA_B200_EINVAL, "%s: dst_uv is for NV12 only, or I420, YUV444, P010, YUV420P10, YUV444P10, YUV422P, "
                    "YUV422P10, YUVA420P and YUVA444P10: %s has no chroma plane", who,
                    format_name(desc->format));
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    for (int i = 0; i < count; ++i) {
        if (streams[i] < 0 || streams[i] >= v.batch)
            return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, streams[i], v.batch);
        if ((rc = dst_check(v, dst[i], "dst", i, who)) != 0) return rc;
        if (dst_uv && (rc = dst_check(v, dst_uv[i], "dst_uv", i, who)) != 0) return rc;
    }
    return 0;
}

// On the handle's stream, where readback copies: after the latest raster pass, before the next one can overwrite a slot
int export_run(ExportKind kind, glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
               const glava_b200_export* desc, const glava_b200_export_scale* scale, void* after_event, void* done_event,
               const uint8_t* opacity, const char* who) {
    clear_error();
    if (!who) who = kCallName[(int) kind];
    if (!r || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_export_scale q;
    int rc = export_check(kind, r, streams, count, dst, dst_uv, desc, scale, who, &q);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    if (kind == ExportKind::overlay) {
        const size_t fb_bytes = (size_t) v.slots * (size_t) v.h * (size_t) v.w * 4;
        if ((rc = overlay_geometry_check(v.w, v.h, count, dst, dst_uv, *desc, &v.fb, &fb_bytes, 1, who)) != 0) return rc;
    }
    const bool yuv = export_ycbcr(desc->format), planes = export_chroma_planes(desc->format);
    // the alpha formats run under their kernel format code, composited only under any other opacity than native
    const bool alpha = export_yuva(desc->format) || (desc->flags & GLAVA_B200_EXPORT_STRAIGHT);
    const int over = alpha ? !v.native : yuv || (desc->flags & GLAVA_B200_EXPORT_OVER) ? 1 : 0;
    const ExportPlanes pl = export_planes(desc->format, desc->pitch, desc->uv_offset, q.out_h);
    CU(cudaSetDevice(v.device));
    // the overlay's opacity (DESIGN 4.20): the fade kernel unless every K is 255, K = 0 entries left out of the list
    const bool fade = opacity_fades(opacity, count);
    int n = 0;
    for (int i = 0; i < count; ++i) n += !fade || opacity[i] ? 1 : 0;
    // export_kernel's entries have no chroma pointer (its machine code stays as measured); the others carry one per entry
    const size_t bytes = (size_t) n * (kind == ExportKind::frames ? sizeof(ExportEntry) : sizeof(ExportEntryUV));
    ExportList* L = nullptr;
    if ((rc = list_room(v, bytes, &L)) != 0) return rc;
    CU(cudaEventSynchronize(L->ev[L->cur]));                // the copy that last read h[cur] (four calls ago)
    uint8_t* const host = L->h[L->cur];
    for (int i = 0, k = 0; i < count; ++i) {
        if (fade && !opacity[i]) continue;
        uint8_t* const d = (uint8_t*) dst[i];
        const int slot = streams[i] % v.slots;
        const int pad = fade ? opacity[i] : 0;
        if (kind == ExportKind::frames) reinterpret_cast<ExportEntry*>(host)[k++] = { d, slot, 0 };
        else reinterpret_cast<ExportEntryUV*>(host)[k++] = { d, !planes ? nullptr : dst_uv ? (uint8_t*) dst_uv[i] : d + pl.cb, slot, pad };
    }
    count = n;
    return list_enqueue(v, L, bytes, after_event, done_event, [&](const void* d_list) {
        if (kind == ExportKind::frames) {
            ExportArgs a = {};
            common_args(a, v, d_list, count, *desc);
            a.over = over;
            a.bg = background(*desc);
            a.uv_offset = pl.cb;
            a.cr_offset = pl.cr;
            a.enc = export_enc(desc->flags);
            return launch_export(a, v.stream);
        }
        if (kind == ExportKind::scaled) {
            ScaledArgs a = {};
            common_args(a, v, d_list, count, *desc);
            a.over = over;
            a.bg = background(*desc);
            a.src_x = q.src_x; a.src_y = q.src_y; a.src_w = q.src_w; a.src_h = q.src_h; a.out_w = q.out_w; a.out_h = q.out_h;
            const ExportRecip rcp = export_recip((uint64_t) q.src_w * (uint64_t) q.src_h);
            a.div_mul = rcp.mul; a.div_shift = rcp.shift;
            a.cr_offset = pl.cr;
            a.enc = export_enc(desc->flags);
            return launch_export_scaled(a, v.stream);
        }
        OverlayArgs a = {};
        common_args(a, v, d_list, count, *desc);
        a.band = a.native && a.marks && a.mark_rows > 0 ? 1 : 0;   // band items wherever marks exist (DESIGN 4.12)
        a.enc = export_enc(desc->flags);
        a.fade = fade ? 1 : 0;
        return launch_overlay(a, v.stream);
    });
}

}  // namespace glb

extern "C" {

int glava_b200_export_bytes(const glava_b200* r, const glava_b200_export* desc, size_t* bytes) {
    return output_bytes(ExportKind::frames, r, desc, nullptr, bytes, "glava_b200_export_bytes");
}
int glava_b200_export_scaled_bytes(const glava_b200* r, const glava_b200_export* desc, const glava_b200_export_scale* scale,
                                   size_t* bytes) {
    return output_bytes(ExportKind::scaled, r, desc, scale, bytes, "glava_b200_export_scaled_bytes");
}

int glava_b200_export_frames(glava_b200* r, const int* streams, int count, void* const* dst, const glava_b200_export* desc,
                             void* after_event, void* done_event) {
    return export_run(ExportKind::frames, r, streams, count, dst, nullptr, desc, nullptr, after_event, done_event);
}
int glava_b200_export_scaled(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                             const glava_b200_export* desc, const glava_b200_export_scale* scale, void* after_event,
                             void* done_event) {
    return export_run(ExportKind::scaled, r, streams, count, dst, dst_uv, desc, scale, after_event, done_event);
}
int glava_b200_overlay_frames(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                              const glava_b200_export* desc, void* after_event, void* done_event) {
    return export_run(ExportKind::overlay, r, streams, count, dst, dst_uv, desc, nullptr, after_event, done_event);
}
int glava_b200_overlay_frames_opacity(glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                                      const glava_b200_export* desc, const uint8_t* opacity, void* after_event, void* done_event) {
    return export_run(ExportKind::overlay, r, streams, count, dst, dst_uv, desc, nullptr, after_event, done_event, opacity,
                      "glava_b200_overlay_frames_opacity");
}

}  // extern "C"
