// export_ladder.cpp — the host half of glava_b200_export_ladder (DESIGN 4.13): every rung checked by export.cpp's
// export_check as a scaled export that names the rung, the schedule of ladder_plan.h built once per geometry and kept on
// the device, one [count][nrungs] list and one launch of export_ladder_kernel (export_kernels.cu) through export_list.h's
// enqueue.  Kept apart from export.cpp so that the other exports build and link without the ladder's launcher.
#include "internal.h"
#include "export_core.h"
#include "export_list.h"
#include "ladder_plan.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <vector>

namespace glb {

int ladder_shape_check(const glava_b200_export_rung* rungs, int nrungs, const char* who) {
    if (!rungs) return fail(GLAVA_B200_EINVAL, "%s: null rungs", who);
    if (nrungs < 1 || nrungs > GLAVA_B200_LADDER_MAX)
        return fail(GLAVA_B200_EINVAL, "%s: nrungs %d must be 1 to %d", who, nrungs, GLAVA_B200_LADDER_MAX);
    return 0;
}

int ladder_check(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs, int nrungs, void* const* dst,
                 void* const* dst_uv, const char* who, glava_b200_export_scale* q) {
    int rc = ladder_shape_check(rungs, nrungs, who);
    if (rc) return rc;
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    // rung j's destinations, as glava_b200_export_scaled would take them
    std::vector<void*> d((size_t) count), uv((size_t) count);
    for (int j = 0; j < nrungs; ++j) {
        char name[96];
        snprintf(name, sizeof(name), "%s: rung %d", who, j);
        const bool yuv = export_chroma_planes(rungs[j].desc.format);
        for (int i = 0; i < count; ++i) {
            d[i] = dst[(size_t) i * nrungs + j];
            uv[i] = dst_uv ? dst_uv[(size_t) i * nrungs + j] : nullptr;
            if (uv[i] && !yuv)
                return fail(GLAVA_B200_EINVAL, "%s: dst_uv[%d] is for NV12 only, or I420, YUV444, P010, YUV420P10, YUV444P10, "
                            "YUV422P, YUV422P10, YUVA420P and YUVA444P10 (entry %d)", name,
                            i * nrungs + j, i);
        }
        rc = export_check(ExportKind::scaled, r, streams, count, d.data(), dst_uv && yuv ? uv.data() : nullptr, &rungs[j].desc,
                          &rungs[j].scale, name, q ? q + j : nullptr);
        if (rc) return rc;
    }
    return 0;
}

// What zero pixels become in a rung under encoding E: NV12's zy / zuv into g, and export_zero (planar 10-bit: export_zero10;
// 4:2:2: export_zero422; the alpha formats: export_zero_alpha) for the other formats
template <int E>
static ExportZeroA rung_zero(const ExportFmt& f, LadderRung* g) {
    const uint32_t zero4[4] = { 0u, 0u, 0u, 0u };
    uint32_t zy1;
    g->zuv = export_nv12_quad<E>(f, zero4, zero4, &g->zy, &zy1);
    if (export_alpha(f.format)) return export_zero_alpha<E>(f);
    const ExportZero z = export_422(f.format) ? export_zero422<E>(f) : export_p10(f.format) ? export_zero10<E>(f) : export_zero<E>(f);
    return { z.y, z.u, z.v, 0u };
}

// the device schedule for `geom`, built and uploaded on the raster stream when the geometry differs from the last ladder's
static int ladder_schedule_room(const RendererView& v, ExportList* L, const LadderGeom* geom, int nrungs, uint32_t* units) {
    std::vector<int> key = { v.w, v.h, nrungs };
    for (int j = 0; j < nrungs; ++j) {
        const LadderGeom& g = geom[j];
        key.insert(key.end(), { g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h, (int) g.whole, (int) g.pairs });
    }
    if (key == L->sched_key && L->sched_cap) { *units = (uint32_t) L->sched_h.size(); return 0; }
    L->sched_key.clear();
    cudaStream_t st = (cudaStream_t) v.stream;
    CU(cudaStreamSynchronize(st));                          // a ladder still running reads the old schedule and sched_h
    L->sched_h = ladder_schedule(v.w, v.h, geom, nrungs);
    const size_t bytes = L->sched_h.size() * sizeof(uint64_t);
    if (bytes > L->sched_cap) {
        L->sched_cap = 0;
        int rc;
        if ((rc = L->sched.alloc(bytes)) != 0) return rc;
        L->sched_cap = bytes;
    }
    CU(cudaMemcpyAsync(L->sched, L->sched_h.data(), bytes, cudaMemcpyHostToDevice, st));
    L->sched_key = key;
    *units = (uint32_t) L->sched_h.size();
    return 0;
}

int ladder_run(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs, int nrungs, void* const* dst,
               void* const* dst_uv, void* after_event, void* done_event, const char* who) {
    clear_error();
    if (!r) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_export_scale q[GLAVA_B200_LADDER_MAX];
    int rc = ladder_check(r, streams, count, rungs, nrungs, dst, dst_uv, who, q);
    if (rc) return rc;
    const RendererView v = renderer_view(r);
    LadderGeom geom[GLAVA_B200_LADDER_MAX];
    ExportPlanes planes[GLAVA_B200_LADDER_MAX];
    for (int j = 0; j < nrungs; ++j) {
        const glava_b200_export& d = rungs[j].desc;
        geom[j] = { q[j].src_x, q[j].src_y, q[j].src_w, q[j].src_h, q[j].out_w, q[j].out_h, false, export_420(d.format) };
        geom[j].whole = ladder_whole(v.w, v.h, geom[j]);
        planes[j] = export_planes(d.format, d.pitch, d.uv_offset, q[j].out_h);
    }
    CU(cudaSetDevice(v.device));
    const size_t n = (size_t) count * (size_t) nrungs, bytes = n * sizeof(ExportEntryUV);
    ExportList* L = nullptr;
    if ((rc = list_room(v, bytes, &L)) != 0) return rc;
    uint32_t units = 0;
    if ((rc = ladder_schedule_room(v, L, geom, nrungs, &units)) != 0) return rc;
    CU(cudaEventSynchronize(L->ev[L->cur]));                // the copy that last read h[cur] (four calls ago)
    ExportEntryUV* const host = reinterpret_cast<ExportEntryUV*>((uint8_t*) L->h[L->cur]);
    for (int i = 0; i < count; ++i) {
        const int slot = streams[i] % v.slots;
        for (int j = 0; j < nrungs; ++j) {
            const size_t e = (size_t) i * nrungs + j;
            uint8_t* const d = (uint8_t*) dst[e];
            uint8_t* const uv = !export_chroma_planes(rungs[j].desc.format) ? nullptr : dst_uv ? (uint8_t*) dst_uv[e] : d + planes[j].cb;
            host[e] = { d, uv, slot, 0 };
        }
    }
    return list_enqueue(v, L, bytes, after_event, done_event, [&](const void* d_list) {
        LadderArgs a = {};
        a.fb = v.fb;
        a.marks = v.mark_key ? v.marks : nullptr;           // as common_args
        a.mark_rows = v.mark_key >> 2;
        a.list = static_cast<const ExportEntryUV*>(d_list); a.count = count; a.w = v.w; a.h = v.h;
        a.native = v.native; a.nrungs = nrungs;
        a.sched = L->sched; a.units = units;
        for (int j = 0; j < nrungs; ++j) {
            const glava_b200_export& d = rungs[j].desc;
            LadderRung& g = a.rung[j];
            g.format = export_kernel_format(d.format, d.flags);
            // the alpha formats are composited only under any other opacity than native (export.cpp export_run)
            g.over = export_alpha(g.format) ? !v.native : export_ycbcr(d.format) || (d.flags & GLAVA_B200_EXPORT_OVER) ? 1 : 0;
            g.whole = geom[j].whole ? 1 : 0;
            g.bg = background(d);
            g.pitch = d.pitch;
            g.src_x = q[j].src_x; g.src_y = q[j].src_y; g.src_w = q[j].src_w; g.src_h = q[j].src_h;
            g.out_w = q[j].out_w; g.out_h = q[j].out_h;
            const ExportRecip rcp = export_recip((uint64_t) q[j].src_w * (uint64_t) q[j].src_h);
            g.div_mul = rcp.mul; g.div_shift = rcp.shift;
            g.enc = export_enc(d.flags);
            // what a zero pixel becomes, as export_kernel and export_scaled_kernel compute it before their loops
            const ExportFmt f = { g.format, g.over, v.native, g.bg };
            g.zpx = export_px(f, 0u);
            g.zc = f.over ? export_over(0u, f.bg, f.native) : 0u;
            // NV12's words, and the other Y'CbCr formats' as export_yuv_kernel / export_p10_kernel compute them, in the
            // rung's encoding
            ExportZeroA z;
            switch (g.enc) {
            case 1: z = rung_zero<1>(f, &g); break;
            case 2: z = rung_zero<2>(f, &g); break;
            case 3: z = rung_zero<3>(f, &g); break;
            case GLB_ENC_PQ: z = rung_zero<GLB_ENC_PQ>(f, &g); break;
            case GLB_ENC_HLG: z = rung_zero<GLB_ENC_HLG>(f, &g); break;
            default: z = rung_zero<0>(f, &g); break;
            }
            a.yuv[j] = { planes[j].cr, z.y, z.u, z.v, z.a };
        }
        return launch_export_ladder(a, v.stream);
    });
}
}  // namespace glb

extern "C" int glava_b200_export_ladder(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs,
                                        int nrungs, void* const* dst, void* const* dst_uv, void* after_event, void* done_event) {
    return glb::ladder_run(r, streams, count, rungs, nrungs, dst, dst_uv, after_event, done_event, "glava_b200_export_ladder");
}
