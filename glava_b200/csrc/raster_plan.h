// raster_plan.h — the launch of one raster pass, chosen in one place (host only).
//
// The raster half of an update runs one of eleven kernels and template instantiations (DESIGN 4.2), with a tile shape, an
// optional column table (graph / wave) or per-stream texture min / max (circle) in front of it, in chunks of streams, and
// with or without dirty-row marks.  raster_tables decides which audio-independent tables capi.cu build_tables makes;
// plan_raster makes every other choice from the parameters the raster launch sees (raster_view), the tables that exist and
// the environment overrides (RasterKnobs).  run_update computes the plan at every raster pass and launch_raster executes it.
// No CUDA here: tests/emul compiles the same decision for the host test tier.
#ifndef GLB_RASTER_PLAN_H
#define GLB_RASTER_PLAN_H

#include "raster_core.h"

#include <cmath>
#include <cstddef>
#include <cstdlib>

namespace glb {

#define RADIAL_MAX_BARS 1024     // bar heights raster_radial_geo_kernel keeps in shared memory

// ---- environment overrides (GLAVA_B200_<name>, DESIGN 6.2) ------------------------------------------------------------
struct RasterKnobs {
    int  rows = 0;              // ROWS: rows per CTA (0: the kernel's default)
    int  bx = 0;                // BX: threads per CTA, a multiple of 32 in [32, 256] (0: by the frame width)
    int  gw_minb = 4;           // GW_MINB=5: graph / wave with the column table at <= 48 registers (5 CTAs of 256) instead of 64
    int  circle_tiles = 16;     // CIRCLE_TILES: 128 x 8 tiles per circle CTA (128 rows)
    bool full_store = false;    // FULL_STORE (non-zero): the bars / graph / wave rasters ignore their dirty-row marks
    bool no_coltab = false;     // NO_COLTAB: graph / wave sample their columns in the raster kernel
    bool no_texmm = false;      // NO_TEXMM: circle without the per-stream annulus
    bool no_geo = false;        // NO_GEO: no polar geometry cache (read when the tables are built)
    bool ctile = false;         // CTILE: the circle tile cull (read when the tables are built)
};

// `get(name)`: the value of the variable GLAVA_B200_<...> or nullptr (getenv in the library, a dictionary in the host build).
// A value outside a knob's range leaves its default.
template <class Get>
RasterKnobs raster_knobs(Get get) {
    RasterKnobs k;
    const char* e;
    if ((e = get("GLAVA_B200_ROWS"))) { const int v = atoi(e); if (v > 0) k.rows = v; }
    if ((e = get("GLAVA_B200_BX"))) { const int v = atoi(e); if (v >= 32 && v <= 256 && v % 32 == 0) k.bx = v; }
    if ((e = get("GLAVA_B200_GW_MINB"))) k.gw_minb = atoi(e) == 5 ? 5 : 4;
    if ((e = get("GLAVA_B200_CIRCLE_TILES"))) { const int v = atoi(e); if (v > 0) k.circle_tiles = v; }
    if ((e = get("GLAVA_B200_FULL_STORE"))) k.full_store = atoi(e) != 0;
    k.no_coltab = get("GLAVA_B200_NO_COLTAB") != nullptr;
    k.no_texmm = get("GLAVA_B200_NO_TEXMM") != nullptr;
    k.no_geo = get("GLAVA_B200_NO_GEO") != nullptr;
    k.ctile = get("GLAVA_B200_CTILE") != nullptr;
    return k;
}

// ---- audio-independent tables ------------------------------------------------------------------------------------------
// radial and circle spend almost all their arithmetic (atan, sqrt, sin, mod, colour ramp, blending, premultiply) on
// quantities that depend on the pixel position and the parameters only.  They are evaluated ONCE per renderer over the
// bounding box of the disc that can be non-zero (polar_geo_kernel, the same core functions, so nothing changes numerically)
// and every frame of every stream reuses them out of L2.  box = {x0, y0, w, h} (x0, w multiples of 4); returns the bytes
// of the cache (0: the module has none, or the disc misses the frame).
inline size_t polar_geo_box(const glava_b200_params& p, int box[4]) {
    float reach, cx, cy;
    if (p.module == GLAVA_B200_MOD_RADIAL) { reach = radial_reach(p); cx = (float) (p.w / 2) - p.radial_off_x; cy = (float) (p.h / 2) - p.radial_off_y; }
    else if (p.module == GLAVA_B200_MOD_CIRCLE) { reach = circle_reach(p); cx = (float) (p.w / 2); cy = (float) (p.h / 2); }
    else { box[0] = box[1] = box[2] = box[3] = 0; return 0; }
    const int wpad = (p.w + 3) & ~3;
    int x0 = (int) floorf(cx - reach) - 3, x1 = (int) ceilf(cx + reach) + 4;
    int y0 = (int) floorf(cy - reach) - 3, y1 = (int) ceilf(cy + reach) + 4;
    x0 = x0 < 0 ? 0 : (x0 & ~3); x1 = x1 > wpad ? wpad : ((x1 + 3) & ~3);
    y0 = y0 < 0 ? 0 : y0; y1 = y1 > p.h ? p.h : y1;
    if (x1 <= x0 || y1 <= y0) { box[0] = box[1] = box[2] = box[3] = 0; return 0; }
    box[0] = x0; box[1] = y0; box[2] = x1 - x0; box[3] = y1 - y0;
    // radial: [full 16 B/px][{lit, dR} 8 B/px][class code 1 B/px]; circle: 16 B/px
    const size_t px = (size_t) box[2] * box[3];
    return p.module == GLAVA_B200_MOD_RADIAL ? px * 25 : px * 16;
}

struct RasterTables {
    bool   geo = false;            // the polar geometry cache
    int    box[4] = { 0, 0, 0, 0 };  // its box (polar_geo_box)
    size_t geo_bytes = 0;          // of one cache
    bool   ctile = false;          // circle: the per-tile texel reference ranges (launch_circle_tiles), built from the cache
    int    style_slots = 1;        // style slots (DESIGN 4.9); more than slot 0 ("no override") selects the styled kernels
    int    geo_caches = 1;         // radial: one cache per distinct (fg, bg) pair of the slots; circle: always one
};

// p: the effective parameters (not the raster view: the tables follow what the K5 pass really did), with the largest
// |AMPLIFY| of the style slots (style_reach_params), so that the box holds every slot's disc.  style_slots / geo_caches:
// the slots and the radial caches they need; all caches together stay within the 512 MiB of a single one, else the
// per-pixel radial kernel runs, as for a box that is too big.
inline RasterTables raster_tables(const glava_b200_params& p, const RasterKnobs& k, int style_slots = 1, int geo_caches = 1) {
    RasterTables t;
    t.style_slots = style_slots;
    t.geo_caches = p.module == GLAVA_B200_MOD_RADIAL ? geo_caches : 1;
    // circle: only when the module samples a pre-smoothed texture, i.e. smooth_audio() is a single texelFetch
    if (p.module == GLAVA_B200_MOD_RADIAL || (p.module == GLAVA_B200_MOD_CIRCLE && p.smooth_pass)) {
        // radial caches lie back to back, `geo_bytes` apart: a box of w x h pixels takes 25 B per pixel, so the stride is
        // rounded up to 256 B, else cache 1 of a box whose w * h is not a multiple of 16 starts off the 16-byte alignment
        // of its int4 entries
        const size_t bytes = (polar_geo_box(p, t.box) + 255) & ~(size_t) 255;
        t.geo = bytes > 0 && bytes * (size_t) t.geo_caches <= ((size_t) 512 << 20) && !k.no_geo;
        t.geo_bytes = t.geo ? bytes : 0;
        // per-tile annulus from bucketed texture min / max (DESIGN 4.2): off by default, GLAVA_B200_CTILE=1 enables it (the
        // curve's halo keeps most tiles of the annulus alive and every live tile pays the bucket reduction)
        t.ctile = t.geo && p.module == GLAVA_B200_MOD_CIRCLE && k.ctile;
    }
    return t;
}

// params.shader_pre_smoothed: the module's stage-1 shader believes something else about its textures than what the K5 pass
// did.  Only the raster launch sees that belief (as its smooth_pass); everything before it follows the real one.
inline glava_b200_params raster_view(const glava_b200_params& p) {
    glava_b200_params v = p;
    if (p.shader_pre_smoothed) v.smooth_pass = p.shader_pre_smoothed == 1 ? 1 : 0;
    return v;
}

// ---- the plan -----------------------------------------------------------------------------------------------------------
enum class RasterKernel {
    GENERIC,        // raster_generic_kernel: every pixel through module_px (any option, any opacity)
    BARS,           // raster_bars_kernel
    GRAPH,          // raster_graph_kernel<false, 1>: columns sampled in the kernel
    GRAPH_TAB4,     // raster_graph_kernel<true, 4>: columns from the column table
    GRAPH_TAB5,     // raster_graph_kernel<true, 5>
    WAVE,           // raster_wave_kernel<false, 1>
    WAVE_TAB4,      // raster_wave_kernel<true, 4>
    WAVE_TAB5,      // raster_wave_kernel<true, 5>
    RADIAL,         // raster_radial_kernel: per-pixel polar maths
    RADIAL_GEO,     // raster_radial_geo_kernel: from the geometry cache
    CIRCLE,         // raster_circle_kernel (with or without the cache)
};

struct RasterPlan {
    RasterKernel kernel = RasterKernel::GENERIC;
    int  bx = 128;              // threads per CTA (circle: 256)
    int  rows = 8;              // rows per CTA (not circle)
    int  minb = 0;              // graph / wave: the instantiation's register budget (__launch_bounds__(256, minb))
    int  circle_tiles = 0;      // circle: 128 x 8 tiles per CTA
    bool coltab = false;        // column_table_kernel runs before the raster kernel (RasterArgs::coltab)
    bool texmm = false;         // texmm_kernel runs before the raster pass (RasterArgs::texmm)
    bool ctile = false;         // the circle tile cull (RasterArgs::ctile)
    bool rowtab = false;        // RasterArgs::rowtab is passed
    bool geo = false;           // RasterArgs::geo is passed
    int  chunk = 1;             // streams per launch
    int  mark_key = 0;          // the dirty-row marks' layout the kernel reads and writes (0: it keeps none)
    int  launches = 0;          // kernel launches of the pass, texmm_kernel included
    bool styled = false;        // the styled instantiation of the kernels (RasterArgs::style_of / styles are passed)
};

// threads per row-segment: prefer an exact tiling of w / 4
inline int pick_block_x(int quads) {
    static const int cand[] = { 96, 160, 128, 192, 256, 64 };
    for (int c : cand) if (quads % c == 0) return c;
    return 128;
}

// v: the raster view (raster_view); t: the tables that exist; slots: framebuffer slots.
inline RasterPlan plan_raster(const glava_b200_params& v, const RasterTables& t, int batch, int slots, const RasterKnobs& k) {
    RasterPlan pl;
    const int m = v.module;
    pl.rowtab = m == GLAVA_B200_MOD_BARS || m == GLAVA_B200_MOD_GRAPH;
    pl.geo = t.geo && !(m == GLAVA_B200_MOD_CIRCLE && v.shader_pre_smoothed);   // the circle cache is laid out for the consistent case
    pl.texmm = m == GLAVA_B200_MOD_CIRCLE && pl.geo && !k.no_texmm;
    pl.ctile = pl.texmm && t.ctile;
    // The specialised kernels assume native opacity (a fragment left at vec4(0) stores 0, whole zero rows / discs are skipped);
    // with GL blending (premultiply_alpha == 0) every stage output is blended over the clear colour: generic kernel.
    const bool native = v.premultiply_alpha != 0;
    const bool bars  = native && m == GLAVA_B200_MOD_BARS && !v.bars_mirror_yx && (v.w & 3) == 0;
    const bool graph = native && m == GLAVA_B200_MOD_GRAPH && !v.graph_join_channels && !v.graph_anti_alias;
    const bool wave  = native && m == GLAVA_B200_MOD_WAVE;
    const bool rgeo  = native && m == GLAVA_B200_MOD_RADIAL && pl.geo && v.radial_nbars <= RADIAL_MAX_BARS
                       && !(v.radial_bar_outline_width > 0.0f);      // the cache holds two values per pixel, the end cap needs three
    const bool wide = bars || graph || wave;                         // __launch_bounds__(256); the others take at most 128 threads
    pl.coltab = (graph || wave) && !k.no_coltab;
    pl.minb = (graph || wave) ? (pl.coltab ? k.gw_minb : 1) : 0;
    if (bars) pl.kernel = RasterKernel::BARS;
    else if (graph) pl.kernel = !pl.coltab ? RasterKernel::GRAPH : (pl.minb == 5 ? RasterKernel::GRAPH_TAB5 : RasterKernel::GRAPH_TAB4);
    else if (wave) pl.kernel = !pl.coltab ? RasterKernel::WAVE : (pl.minb == 5 ? RasterKernel::WAVE_TAB5 : RasterKernel::WAVE_TAB4);
    else if (rgeo) pl.kernel = RasterKernel::RADIAL_GEO;
    else if (native && m == GLAVA_B200_MOD_RADIAL) pl.kernel = RasterKernel::RADIAL;
    else if (native && m == GLAVA_B200_MOD_CIRCLE) pl.kernel = RasterKernel::CIRCLE;
    // rows per CTA.  bars: with the dirty-row marks a band above the bars stores nothing but still pays the per-column set-up, so
    // taller bands win.  On an H100 SXM (700 W limit), 1080p x 1024 streams, bench steps: 135 / 270 / 360 / 540 / 1080 rows gave
    // 3.60 / 4.66 / 4.81 / 4.87 / 4.94 M frames/s (tools/tune_raster.py); 540 keeps two bands per column for small batches, and
    // 96 / 160 / 256 threads per CTA were within 0.2 % there.  graph / wave pay a per-thread column set-up, so whole columns
    // without the column table; with it their set-up is six loads and short bands win (tools/gw_tune.py sweeps them);
    // radial-from-cache 45.
    pl.rows = bars ? 540 : ((graph || wave) ? (pl.coltab ? (wave ? 16 : 30) : 720) : (rgeo ? 45 : 8));
    if (k.rows) pl.rows = k.rows;
    if (pl.rows > v.h) pl.rows = v.h;
    pl.bx = k.bx ? k.bx : (wide ? pick_block_x((v.w + 3) / 4) : 128);
    if (!wide && pl.bx > 128) pl.bx = 128;
    if (pl.kernel == RasterKernel::CIRCLE) { pl.bx = 256; pl.circle_tiles = k.circle_tiles; }
    // Dirty-row marks.  Their layout depends on the kernel's band height, and a kernel that keeps none (generic, radial, circle)
    // can leave non-zero pixels anywhere: they describe the framebuffer only if the previous launch was the same kernel at the
    // same `rows` (raster_marks_valid).
    pl.mark_key = wide ? ((bars ? 1 : (graph ? 2 : 3)) | (pl.rows << 2)) : 0;
    // One launch covers at most `slots` streams (and at most the grid z limit, 65535): with a framebuffer ring (fb_slots <
    // batch) two streams of one launch must never share a slot, and launches on the same stream are ordered, so slot
    // s % slots ends up holding the highest stream mapped to it.
    pl.chunk = slots < 32768 ? (slots > 0 ? slots : 1) : 32768;
    pl.launches = (pl.texmm ? 1 : 0) + ((batch + pl.chunk - 1) / pl.chunk) * (pl.coltab ? 2 : 1);
    // Styles change no choice above: every kernel reads its stream's slot once per CTA in its styled instantiation, which
    // keeps the marks of the plain one (zero rows do not depend on colours, and AMPLIFY only moves the rows a frame writes)
    pl.styled = t.style_slots > 1;
    return pl;
}

// The module's AMPLIFY field (graph: VSCALE), what a style's `amplify` replaces; nullptr for the test module
inline float* style_amplify_field(glava_b200_params& p) {
    switch (p.module) {
        case GLAVA_B200_MOD_BARS: return &p.bars_amplify;
        case GLAVA_B200_MOD_RADIAL: return &p.radial_amplify;
        case GLAVA_B200_MOD_CIRCLE: return &p.circle_amplify;
        case GLAVA_B200_MOD_GRAPH: return &p.graph_vscale;
        case GLAVA_B200_MOD_WAVE: return &p.wave_amplify;
        default: return nullptr;
    }
}

// What the polar box is built for: p with the largest |AMPLIFY| of the slots' parameters sp[0 .. slots)
inline glava_b200_params style_reach_params(const glava_b200_params& p, const glava_b200_params* sp, int slots) {
    glava_b200_params q = p;
    float* a = style_amplify_field(q);
    if (!a) return q;
    for (int i = 0; i < slots; ++i) {
        glava_b200_params s = sp[i];
        const float v = *style_amplify_field(s);
        if (fabsf(v) > fabsf(*a)) *a = v;
    }
    return q;
}

// Whether the marks describe the framebuffer: the renderer's record `last_key` of the launch that last wrote them (0: none,
// or a kernel that keeps no marks wrote the framebuffer since) is this plan's key.  GLAVA_B200_FULL_STORE=1 stores every
// zero row anyway, for same-process A/B timing.
inline bool raster_marks_valid(const RasterPlan& pl, int last_key, const RasterKnobs& k) {
    return pl.mark_key != 0 && pl.mark_key == last_key && !k.full_store;
}

}  // namespace glb

#endif
