// Host build of the raster plan with stream styles (raster_plan.h), for tests/test_stream_styles.py: what capi.cu
// build_tables and enqueue_raster decide for a renderer whose style slots have the parameters sp[0 .. slots) (sp[0]: the
// renderer's own) and need `geo_caches` radial geometry caches.
#include "../../glava_b200/csrc/raster_plan.h"

#include <cstring>

using namespace glb;

extern "C" {

// out[] = { kernel (RasterKernel), bx, rows, minb, circle_tiles, coltab, texmm, ctile, rowtab, geo, chunk, mark_key, launches,
//           styled, box w, box h, geo_bytes (of one cache), geo_caches }
void emul_styled_raster_plan(const glava_b200_params* sp, int slots, int geo_caches, int batch, int fb_slots,
                             const char* const* names, const char* const* values, int count, long long* out) {
    const RasterKnobs k = raster_knobs([&](const char* name) -> const char* {
        for (int i = 0; i < count; ++i) if (!strcmp(names[i], name)) return values[i];
        return nullptr;
    });
    const RasterTables t = raster_tables(style_reach_params(sp[0], sp, slots), k, slots, geo_caches);
    const RasterPlan pl = plan_raster(raster_view(sp[0]), t, batch, fb_slots, k);
    const long long v[] = { (long long) pl.kernel, pl.bx, pl.rows, pl.minb, pl.circle_tiles, pl.coltab, pl.texmm, pl.ctile,
                            pl.rowtab, pl.geo, pl.chunk, pl.mark_key, pl.launches, pl.styled, t.box[2], t.box[3],
                            (long long) t.geo_bytes, t.geo_caches };
    for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
}

// box[4] = { x0, y0, w, h }: the polar geometry box of a renderer whose style slots have the parameters sp[0 .. slots)
// (polar_geo_box of style_reach_params, as raster_tables builds it); all 0 for the other modules
void emul_styled_geo_box(const glava_b200_params* sp, int slots, int* box) {
    polar_geo_box(style_reach_params(sp[0], sp, slots), box);
}

}  // extern "C"
