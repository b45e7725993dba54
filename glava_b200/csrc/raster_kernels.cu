// raster_kernels.cu — sm_90a kernels of the R16 texture -> RGBA8 framebuffer half of the path:
// one module frame per stream straight into the HBM framebuffer with 128-bit streaming stores, all post
// stages (premultiply, 8-neighbour stencils) fused.   [replaces the module .frag stages of
// shaders/glava/{bars,radial,circle,graph,wave}/ and util/premultiply.frag]
//
// Compiled with --fmad=false: results are bit-identical to the host build of the *_core.h maths.
#include "internal.h"
#include "raster_core.h"
#include "raster_plan.h"

#include <cuda_runtime.h>

namespace glb {

// ---------------------------------------------------------------------------------------------
// raster kernels.  Thread = 4 horizontally adjacent pixels = one 128-bit streaming store.
__device__ __forceinline__ AudioTex make_tex(const glava_b200_params& p, const uint16_t* tex, int stream) {
    AudioTex t;
    t.l = tex + (size_t) (stream * 2) * p.n;
    t.r = t.l + p.n;
    t.n = p.n; t.pre_smoothed = p.smooth_pass; t.sp = smooth_params(p);
    return t;
}
__device__ __forceinline__ void store4(uint32_t* row, int x, int w, const uint32_t px[4]) {
    // rows are 16-byte aligned only when w is a multiple of 4 (x always is)
    if ((w & 3) == 0) __stcs(reinterpret_cast<uint4*>(row + x), make_uint4(px[0], px[1], px[2], px[3]));
    else for (int k = 0; k < 4 && x + k < w; ++k) row[x + k] = px[k];
}

// Rows [ya, yb) of a thread's quad are 0: when the rows are 16-byte aligned this is a bare pointer-increment loop of
// independent 128-bit stores (the compiler unrolls it: several stores in flight per warp), the shape raster_bars_kernel
// reaches the copy peak with.  The same loop written as store4(fb + y * w, ...) keeps a uniform branch on (w & 3) and a
// 64-bit address recomputation around every store — graph / wave are 97 % zero rows and ran at 0.87 / 0.90 with it.
__device__ __forceinline__ void zero_rows(uint32_t* fb, int x, int w, int ya, int yb) {
    if ((w & 3) == 0) {
        const int stride = w >> 2;
        uint4* ptr = reinterpret_cast<uint4*>(fb) + (size_t) ya * stride + (x >> 2);
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 8
        for (int y = ya; y < yb; ++y, ptr += stride) __stcs(ptr, zero);
    } else {
        const uint32_t zero4[4] = { 0u, 0u, 0u, 0u };
        for (int y = ya; y < yb; ++y) store4(fb + (size_t) y * w, x, w, zero4);
    }
}

// Dirty-row mark of the warp that owns the 128-pixel strip of quad x in the band starting at row y0 (RasterArgs::marks).
// Only lane 0 reads and writes it, and no other warp touches it.
__device__ __forceinline__ uint32_t* mark_word(const RasterArgs& a, const glava_b200_params& p, int stream, int x, int y0) {
    return a.marks + ((size_t) (stream % a.slots) * p.h + y0) * ((p.w + 127) >> 7) + (x >> 7);
}
// the rows of [y0, y1) that may be non-zero in memory, as a mark; without valid marks, all of them
__device__ __forceinline__ uint32_t mark_load(const RasterArgs& a, const uint32_t* m, int y0, int y1, unsigned lanes) {
    if (!a.marks_valid) return dirty_pack(y0, y1);
    uint32_t v = 0u;
    if ((threadIdx.x & 31) == 0) v = *m;
    return __shfl_sync(lanes, v, 0);
}
__device__ __forceinline__ void mark_store(uint32_t* m, int lo, int hi) {
    if ((threadIdx.x & 31) == 0) *m = dirty_pack(lo, hi);
}

// Stream styles (DESIGN 4.9).  Every raster kernel has a plain and a styled twin.  The styled one copies its stream's
// StyleSlot (parameters and tables of the slot) into dynamic shared memory once per CTA, before any thread leaves, and reads
// everything through it; the plain one reads the kernel parameter and RasterArgs' tables as it always has.  Six pairs share
// one body: five instantiate a body template, and both radial-from-cache kernels call radial_geo_body with their
// parameters and cache (the kernel's or the slot's).  The plain circle and
// wave kernels keep their own text, because the plain path must stay what it was: moved into a __forceinline__ body that
// takes the chosen `p` as an argument, they compile to other machine code under nvcc 12.9 (tools/sass_diff.py):
// raster_wave_kernel<false, 1> 2968 -> 3040 instructions, raster_circle_kernel 3968 in another schedule.  Passing `a` by
// value, __restrict__ on `a` / `p`, internal linkage and a body instance per kernel do not change that (DESIGN 4.9).  Their
// styled twins repeat that code with the slot's reads; tests/test_gpu_stream_styles.py holds each twin to the plain kernel
// of a batch-1 renderer, frame by frame.
template <bool STYLED>
__device__ __forceinline__ const StyleSlot* stream_style(const RasterStyles& sa, int stream) {
    if constexpr (!STYLED) return nullptr;
    else {
        extern __shared__ int4 style_smem[];
        const int4* src = reinterpret_cast<const int4*>(sa.styles + __ldg(sa.style_of + stream));
        for (int i = threadIdx.x; i < (int) (sizeof(StyleSlot) / sizeof(int4)); i += blockDim.x) style_smem[i] = __ldg(src + i);
        __syncthreads();
        return reinterpret_cast<const StyleSlot*>(style_smem);
    }
}
template <bool STYLED>
__device__ __forceinline__ const glava_b200_params& style_params_of(const StyleSlot* s, const glava_b200_params& p) {
    if constexpr (STYLED) return s->p;
    else return p;
}
#define GLB_STYLED_PAIR(body, bounds, name, styled_name)                                                                        \
    __global__ void bounds name(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int n) {    \
        body<false>(a, p, n, RasterStyles{});                                                                                  \
    }                                                                                                                           \
    __global__ void bounds styled_name(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int n, \
                                       const __grid_constant__ RasterStyles sa) {                                              \
        body<true>(a, p, n, sa);                                                                                                \
    }

// generic: every pixel through module_px() — reference semantics with no hoisting; also the
// fallback for option combinations the specialised kernels do not cover.
template <bool STYLED>
__device__ __forceinline__ void generic_body(const RasterArgs& a, const glava_b200_params& pk, int rows_per_cta, const RasterStyles& sa) {
    const int stream = a.stream0 + blockIdx.z;
    const glava_b200_params& p = style_params_of<STYLED>(stream_style<STYLED>(sa, stream), pk);
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    // polar modules: everything outside a disc around the centre is exactly 0
    // (native opacity only: with blending the far field is the blended clear colour, evaluated per pixel)
    float reach = -1.0f, cx = 0.0f, cy = 0.0f;
    if (!p.premultiply_alpha) { }
    else if (p.module == GLAVA_B200_MOD_RADIAL) { reach = radial_reach(p); cx = (float) (p.w / 2) - p.radial_off_x; cy = (float) (p.h / 2) - p.radial_off_y; }
    else if (p.module == GLAVA_B200_MOD_CIRCLE) { reach = circle_reach(p); cx = (float) (p.w / 2); cy = (float) (p.h / 2); }
    for (int y = y0; y < y1; ++y) {
        uint32_t px[4] = { 0u, 0u, 0u, 0u };
        bool live = true;
        if (reach >= 0.0f) {
            float dy = fabsf((float) y - cy) - 1.0f;
            float dxa = (float) x - cx, dxb = (float) (x + 3) - cx;
            float dxm = (dxa > 0.0f) ? dxa : ((dxb < 0.0f) ? -dxb : 0.0f);   // distance of the 4-pixel span from cx
            dxm -= 1.0f;
            if (dy < 0.0f) dy = 0.0f;
            if (dxm < 0.0f) dxm = 0.0f;
            live = (dxm * dxm + dy * dy) <= reach * reach;
        }
        if (live) {
#pragma unroll
            for (int k = 0; k < 4; ++k) if (x + k < p.w) px[k] = module_px(p, t, x + k, y);
        }
        store4(fb + (size_t) y * p.w, x, p.w, px);
    }
}
GLB_STYLED_PAIR(generic_body, __launch_bounds__(128), raster_generic_kernel, raster_generic_styled_kernel)

// bars (default orientation): column state in registers, row colours from a per-renderer table
__device__ __forceinline__ void bars_rowtab_body(uint2* __restrict__ tab, const glava_b200_params& p) {
    int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= p.h) return;
    if (p.module == GLAVA_B200_MOD_GRAPH) {
        const uint32_t c = graph_row(p, y);
        const uint32_t cm = y > 0 ? graph_row(p, y - 1) : 0u, cp = (y + 1 < p.h) ? graph_row(p, y + 1) : 0u;
        tab[y] = make_uint2(c, (((c & cm & cp) >> 24) == 255u) ? 1u : 0u);     // .y: rows y-1, y, y+1 all have alpha 1
        return;
    }
    float fy = (float) y + 0.5f;
    float d = p.bars_flip ? (float) p.h - fy : fy;
    BarsRow r = bars_row(p, d);
    tab[y] = make_uint2(r.fill, r.outl);
}
__global__ void bars_rowtab_kernel(uint2* __restrict__ tab, const __grid_constant__ glava_b200_params p) {
    bars_rowtab_body(tab, p);
}
int launch_bars_rowtab(const glava_b200_params& p, void* d_rowtab, void* stream) {
    bars_rowtab_kernel<<<(p.h + 127) / 128, 128, 0, (cudaStream_t) stream>>>(reinterpret_cast<uint2*>(d_rowtab), p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "bars rowtab kernel launch: %s", cudaGetErrorString(e));
    return 0;
}
// Rows are addressed by t = distance from the bars' base line (t = y, or h-1-y with FLIP), for which
// d = t + 0.5 exactly in float.  `d < lim` / `d <= lim` are monotone in t, so each column's two float
// compares per pixel collapse into two integer row thresholds computed once (and corrected with the
// exact float predicate, so the result is bit-identical to evaluating bars/1.frag per pixel).
__device__ __forceinline__ int bars_rows_below(float lim, bool inclusive, int h) {
    float e = ceilf(lim - 0.5f);
    int t = (e > 0.0f) ? ((e < (float) h) ? (int) e : h) : 0;
    while (t > 0 && !(inclusive ? ((float) (t - 1) + 0.5f <= lim) : ((float) (t - 1) + 0.5f < lim))) --t;
    while (t < h && (inclusive ? ((float) t + 0.5f <= lim) : ((float) t + 0.5f < lim))) ++t;
    return t;
}

// requires w % 4 == 0 (128-bit row alignment) and MIRROR_YX == 0
template <bool STYLED>
__device__ __forceinline__ void bars_body(const RasterArgs& a, const glava_b200_params& pk, int rows_per_cta, const RasterStyles& sa) {
    const int stream = a.stream0 + blockIdx.z;
    const StyleSlot* const sty = stream_style<STYLED>(sa, stream);
    const glava_b200_params& p = style_params_of<STYLED>(sty, pk);
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if ((x & ~127) >= p.w) return;                                        // the whole warp is right of the frame
    const bool valid = x < p.w;
    const AudioTex t = make_tex(p, a.tex, stream);
    const uint2* __restrict__ rowtab = reinterpret_cast<const uint2*>(STYLED ? sty->rowtab : a.rowtab);
    const bool has_outline = p.bars_outline_width > 0.0f;
    int ya[4], yb[4]; bool inner[4];
    int tmax = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        BarsCol c = { 0, 0.0f, 0.0f };
        if (valid) c = bars_column(p, t, (float) (x + k) + 0.5f, p.w);
        inner[k] = c.cls == 1;
        ya[k] = c.cls ? bars_rows_below(c.vm, false, p.h) : 0;          // t <  ya : d <  v - outline  -> COLOR / BAR_OUTLINE by column
        yb[k] = (c.cls && has_outline) ? bars_rows_below(c.v, true, p.h) : 0;   // t <  yb : d <= v            -> BAR_OUTLINE
        tmax = max(tmax, max(ya[k], yb[k]));
    }
    tmax = __reduce_max_sync(0xffffffffu, tmax);                          // rows t >= tmax are 0 for the whole warp
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    const int stride = p.w >> 2;
    uint4* const base = reinterpret_cast<uint4*>(a.fb) + (size_t) (stream % a.slots) * stride * p.h + (x >> 2);
    // split the band into the rows that can hold bar pixels and the all-zero rest
    int f0, f1, z0, z1;
    if (!p.bars_flip) { f0 = y0; f1 = min(y1, tmax); z0 = max(y0, tmax); z1 = y1; }
    else              { z0 = y0; z1 = min(y1, p.h - tmax); f0 = max(y0, p.h - tmax); f1 = y1; }
    uint32_t* const mark = mark_word(a, p, stream, x, y0);
    {   // of the zero rows, only those the previous frame in this slot may have left non-zero
        int s0, s1;
        dirty_zero_span(mark_load(a, mark, y0, y1, 0xffffffffu), z0, z1, &s0, &s1);
        uint4* ptr = base + (size_t) s0 * stride;
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
        for (int y = s0; y < s1; ++y, ptr += stride) if (valid) __stcs(ptr, zero);
    }
    mark_store(mark, f0, f1);
    {
        uint4* ptr = base + (size_t) f0 * stride;
        for (int y = f0; y < f1; ++y, ptr += stride) {
            const uint2 rc = __ldg(&rowtab[y]);
            const int tt = p.bars_flip ? (p.h - 1 - y) : y;
            uint32_t px[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) px[k] = (tt < ya[k]) ? (inner[k] ? rc.x : rc.y) : ((tt < yb[k]) ? rc.y : 0u);
            if (valid) __stcs(ptr, make_uint4(px[0], px[1], px[2], px[3]));
        }
    }
}
GLB_STYLED_PAIR(bars_body, __launch_bounds__(256), raster_bars_kernel, raster_bars_styled_kernel)

// graph: heights of 6 columns in registers, row colours from a per-renderer table.  Pixels whose whole
// 3x3 neighbourhood is filled (or empty) skip the stencil — exact, because then avg.a is exactly the
// row alpha (or 0) and graph/2.frag changes nothing.  Without INVERT the fill test `y + 1.5 <= s` is
// monotone in y, so a warp's band splits into [full | plain row-colour copy | full (edge band) | zero]
// with warp-uniform integer row bounds; only the edge band pays for the stencil.
__device__ __forceinline__ int graph_first_row(float lim, int off, int h) {
    // first y in [0, h] for which row y + off is NOT filled against height `lim`: (float)(y + off) + 1.5f > lim
    // (graph/1.frag:116 fills when d + 1.5 <= s); float estimate, then corrected with the exact predicate
    float e = ceilf(lim - 1.5f - (float) off);
    int y = (e > 0.0f) ? ((e < (float) h) ? (int) e : h) : 0;
    while (y > 0 && ((float) (y - 1 + off) + 1.5f > lim)) --y;
    while (y < h && !((float) (y + off) + 1.5f > lim)) ++y;
    return y;
}

// graph / wave: what a column contributes to its pixels depends on the audio through the column alone (graph: the height,
// graph/1.frag:84-114; wave: wave/1.frag:17-31).  One thread per (stream, column) evaluates it once per update into the
// column table; the raster kernels then start with six coalesced loads instead of six dependent texture samples per
// thread and ROW BAND — which had forced whole-column CTAs (1080p: 2560 CTAs of 720 / 360 rows, under two waves).
template <bool WAVE, bool STYLED>
__device__ __forceinline__ void column_table_body(const RasterArgs& a, const glava_b200_params& pk, const RasterStyles& sa) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int stream = a.stream0 + blockIdx.y;
    const glava_b200_params& p = style_params_of<STYLED>(stream_style<STYLED>(sa, stream), pk);
    if (x >= p.w) return;
    const AudioTex t = make_tex(p, a.tex, stream);
    float* ct = a.coltab + (size_t) stream * GLB_COLTAB_PLANES * p.w;
    if (WAVE) {
        const WaveCol c = wave_column(p, t, x);
        ct[x] = c.s; ct[p.w + x] = c.dmin; ct[2 * p.w + x] = c.dmax; ct[3 * p.w + x] = c.thick; ct[4 * p.w + x] = __uint_as_float(c.color);
    } else ct[x] = graph_height(p, t, x);
}
template <bool WAVE>
__global__ void __launch_bounds__(128)
column_table_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p) {
    column_table_body<WAVE, false>(a, p, RasterStyles{});
}
template <bool WAVE>
__global__ void __launch_bounds__(128)
column_table_styled_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p,
                           const __grid_constant__ RasterStyles sa) {
    column_table_body<WAVE, true>(a, p, sa);
}

template <bool TAB, bool STYLED>
__device__ __forceinline__ void graph_body(const RasterArgs& a, const glava_b200_params& pk, int rows_per_cta, const RasterStyles& sa) {
    const int stream = a.stream0 + blockIdx.z;
    const StyleSlot* const sty = stream_style<STYLED>(sa, stream);
    const glava_b200_params& p = style_params_of<STYLED>(sty, pk);
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    float s[6];                                        // columns x-1 .. x+4
    const float* __restrict__ ct = TAB ? a.coltab + (size_t) stream * GLB_COLTAB_PLANES * p.w : nullptr;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        int xc = x - 1 + k;
        s[k] = (xc >= 0 && xc < p.w) ? (TAB ? __ldg(ct + xc) : graph_height(p, t, xc)) : 0.0f;
    }
    float lo[4], hi[4]; bool inner_x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        lo[k] = fminf(s[k], fminf(s[k + 1], s[k + 2]));
        hi[k] = fmaxf(s[k], fmaxf(s[k + 1], s[k + 2]));
        inner_x[k] = (x + k - 1 >= 0) && (x + k + 1 < p.w);
    }
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    const uint2* __restrict__ rowtab = reinterpret_cast<const uint2*>(STYLED ? sty->rowtab : a.rowtab);   // [h] {graph_row(y), rows y-1..y+1 opaque}

    auto full_rows = [&](int ya, int yb) {             // reference evaluation with per-pixel shortcuts
        for (int y = ya; y < yb; ++y) {
            uint32_t row3[3];
            row3[0] = y > 0 ? __ldg(&rowtab[y - 1]).x : 0u;
            const uint2 rc = __ldg(&rowtab[y]);
            row3[1] = rc.x;
            row3[2] = (y + 1 < p.h) ? __ldg(&rowtab[y + 1]).x : 0u;
            const float dm = graph_d(p, y - 1), dp = graph_d(p, y + 1);
            const float dhi = fmaxf(dm, dp) + 1.5f, dlo = fminf(dm, dp) + 1.5f;   // stage-1 test is d + 1.5 <= s
            const bool inner_y = (y - 1 >= 0) && (y + 1 < p.h);
            const bool opaque = rc.y != 0u;
            uint32_t px[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (dlo > hi[k]) px[k] = 0u;                                              // 3x3 all empty
                else if (dhi <= lo[k] && inner_x[k] && inner_y && opaque) px[k] = row3[1]; // 3x3 all filled, alpha 1
                else {
                    const float s3[3] = { s[k], s[k + 1], s[k + 2] };
                    px[k] = (x + k < p.w) ? graph_px_cols(p, s3, row3, x + k, y) : 0u;
                }
            }
            store4(fb + (size_t) y * p.w, x, p.w, px);
        }
    };

    uint32_t* const mark = mark_word(a, p, stream, x, y0);     // lane 0 is active: lanes past the right edge returned
    if (p.graph_invert > 0) { full_rows(y0, y1); mark_store(mark, y0, y1); return; }

    // thread bounds: rows >= E are empty for all 4 pixels; rows < F (and >= 1, < h-1) are interior for all 4
    int E = 0, F = p.h;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (x + k >= p.w) continue;
        E = max(E, graph_first_row(hi[k], -1, p.h));                 // (y-1)+1.5 > hi  <=> 3x3 empty
        F = min(F, inner_x[k] ? graph_first_row(lo[k], +1, p.h) : 0); // (y+1)+1.5 <= lo <=> 3x3 filled
    }
    const unsigned lanes = __activemask();
    E = __reduce_max_sync(lanes, E); F = __reduce_min_sync(lanes, F);
    const int b1 = min(y1, max(y0, 1));
    const int b2 = max(b1, min(y1, min(F, p.h - 1)));
    const int b3 = max(b2, min(y1, E));
    full_rows(y0, b1);
    for (int y = b1; y < b2; ++y) {
        const uint2 rc = __ldg(&rowtab[y]);
        if (rc.y != 0u) {
            const uint32_t px[4] = { rc.x, x + 1 < p.w ? rc.x : 0u, x + 2 < p.w ? rc.x : 0u, x + 3 < p.w ? rc.x : 0u };
            store4(fb + (size_t) y * p.w, x, p.w, px);
        } else full_rows(y, y + 1);
    }
    full_rows(b2, b3);
    int s0, s1;
    dirty_zero_span(mark_load(a, mark, y0, y1, lanes), b3, y1, &s0, &s1);
    zero_rows(fb, x, p.w, s0, s1);
    mark_store(mark, y0, b3);
}
template <bool TAB, int MINB>
__global__ void __launch_bounds__(256, MINB)
raster_graph_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int rows_per_cta) {
    graph_body<TAB, false>(a, p, rows_per_cta, RasterStyles{});
}
template <bool TAB, int MINB>
__global__ void __launch_bounds__(256, MINB)
raster_graph_styled_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int rows_per_cta,
                         const __grid_constant__ RasterStyles sa) {
    graph_body<TAB, true>(a, p, rows_per_cta, sa);
}

// wave: 6 column descriptors in registers
template <bool TAB, int MINB>
__global__ void __launch_bounds__(256, MINB)
raster_wave_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int rows_per_cta) {
    const int stream = a.stream0 + blockIdx.z;
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    WaveCol c[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        int xc = x - 1 + k;
        xc = xc < 0 ? 0 : (xc >= p.w ? p.w - 1 : xc);   // clamped columns are masked by wave_px_cols
        if (TAB) {
            const float* __restrict__ ct = a.coltab + (size_t) stream * GLB_COLTAB_PLANES * p.w + xc;
            c[k].s = __ldg(ct); c[k].dmin = __ldg(ct + p.w); c[k].dmax = __ldg(ct + 2 * p.w); c[k].thick = __ldg(ct + 3 * p.w);
            c[k].color = __float_as_uint(__ldg(ct + 4 * p.w));
        } else c[k] = wave_column(p, t, xc);
    }
    // rows where any of a pixel's three columns can be lit (+-1 row for the stencil), conservative
    float ylo[4], yhi[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float l = 3.0e38f, h = -3.0e38f;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const WaveCol& w = c[k + j];
            l = fminf(l, fminf(w.s - w.thick, w.s + w.dmin));
            h = fmaxf(h, fmaxf(w.s + w.thick, w.s + w.dmax));
        }
        ylo[k] = l - 2.0f; yhi[k] = h + 2.0f;
    }
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    // rows outside [ra, rb) are 0 for every pixel of this thread: run them as a bare zero-store loop
    float lo4 = fminf(fminf(ylo[0], ylo[1]), fminf(ylo[2], ylo[3])), hi4 = fmaxf(fmaxf(yhi[0], yhi[1]), fmaxf(yhi[2], yhi[3]));
    lo4 = fminf(fmaxf(lo4, -1.0f), 1.0e6f); hi4 = fminf(fmaxf(hi4, -1.0f), 1.0e6f);
    int ra = min(y1, max(y0, (int) floorf(lo4))), rb = max(ra, min(y1, (int) ceilf(hi4) + 1));
    // make the split warp-uniform (lanes past the right edge have already returned)
    const unsigned lanes = __activemask();
    ra = __reduce_min_sync(lanes, ra); rb = __reduce_max_sync(lanes, rb);
    // zero rows on both sides of the line: store those the previous frame in this slot may have left non-zero
    uint32_t* const mark = mark_word(a, p, stream, x, y0);
    const uint32_t old = mark_load(a, mark, y0, y1, lanes);
    int s0, s1;
    dirty_zero_span(old, y0, ra, &s0, &s1);
    zero_rows(fb, x, p.w, s0, s1);
    for (int y = ra; y < rb; ++y) {
        const float fy = (float) y;
        uint32_t px[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (fy < ylo[k] || fy > yhi[k] || x + k >= p.w) { px[k] = 0u; continue; }
            const WaveCol c3[3] = { c[k], c[k + 1], c[k + 2] };
            px[k] = wave_px_cols(p, c3, x + k, y);
        }
        store4(fb + (size_t) y * p.w, x, p.w, px);
    }
    dirty_zero_span(old, rb, y1, &s0, &s1);
    zero_rows(fb, x, p.w, s0, s1);
    mark_store(mark, ra, rb);
}
// styled twin (DESIGN 4.9): the same code reading its stream's style slot
template <bool TAB>
__device__ __forceinline__ void wave_styled_body(const RasterArgs& a, int rows_per_cta, const RasterStyles& sa) {
    const int stream = a.stream0 + blockIdx.z;
    const glava_b200_params& p = stream_style<true>(sa, stream)->p;
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    WaveCol c[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        int xc = x - 1 + k;
        xc = xc < 0 ? 0 : (xc >= p.w ? p.w - 1 : xc);   // clamped columns are masked by wave_px_cols
        if (TAB) {
            const float* __restrict__ ct = a.coltab + (size_t) stream * GLB_COLTAB_PLANES * p.w + xc;
            c[k].s = __ldg(ct); c[k].dmin = __ldg(ct + p.w); c[k].dmax = __ldg(ct + 2 * p.w); c[k].thick = __ldg(ct + 3 * p.w);
            c[k].color = __float_as_uint(__ldg(ct + 4 * p.w));
        } else c[k] = wave_column(p, t, xc);
    }
    // rows where any of a pixel's three columns can be lit (+-1 row for the stencil), conservative
    float ylo[4], yhi[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float l = 3.0e38f, h = -3.0e38f;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const WaveCol& w = c[k + j];
            l = fminf(l, fminf(w.s - w.thick, w.s + w.dmin));
            h = fmaxf(h, fmaxf(w.s + w.thick, w.s + w.dmax));
        }
        ylo[k] = l - 2.0f; yhi[k] = h + 2.0f;
    }
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    // rows outside [ra, rb) are 0 for every pixel of this thread: run them as a bare zero-store loop
    float lo4 = fminf(fminf(ylo[0], ylo[1]), fminf(ylo[2], ylo[3])), hi4 = fmaxf(fmaxf(yhi[0], yhi[1]), fmaxf(yhi[2], yhi[3]));
    lo4 = fminf(fmaxf(lo4, -1.0f), 1.0e6f); hi4 = fminf(fmaxf(hi4, -1.0f), 1.0e6f);
    int ra = min(y1, max(y0, (int) floorf(lo4))), rb = max(ra, min(y1, (int) ceilf(hi4) + 1));
    // make the split warp-uniform (lanes past the right edge have already returned)
    const unsigned lanes = __activemask();
    ra = __reduce_min_sync(lanes, ra); rb = __reduce_max_sync(lanes, rb);
    // zero rows on both sides of the line: store those the previous frame in this slot may have left non-zero
    uint32_t* const mark = mark_word(a, p, stream, x, y0);
    const uint32_t old = mark_load(a, mark, y0, y1, lanes);
    int s0, s1;
    dirty_zero_span(old, y0, ra, &s0, &s1);
    zero_rows(fb, x, p.w, s0, s1);
    for (int y = ra; y < rb; ++y) {
        const float fy = (float) y;
        uint32_t px[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (fy < ylo[k] || fy > yhi[k] || x + k >= p.w) { px[k] = 0u; continue; }
            const WaveCol c3[3] = { c[k], c[k + 1], c[k + 2] };
            px[k] = wave_px_cols(p, c3, x + k, y);
        }
        store4(fb + (size_t) y * p.w, x, p.w, px);
    }
    dirty_zero_span(old, rb, y1, &s0, &s1);
    zero_rows(fb, x, p.w, s0, s1);
    mark_store(mark, ra, rb);
}
template <bool TAB, int MINB>
__global__ void __launch_bounds__(256, MINB)
raster_wave_styled_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params, int rows_per_cta,
                         const __grid_constant__ RasterStyles sa) {
    wave_styled_body<TAB>(a, rows_per_cta, sa);
}

// circle: stage 1 (polar line test) is evaluated once per pixel of a tile + 1-pixel halo into shared
// memory, then stages 2 (8-neighbour fill-in) and 3 (premultiply) read the tile.  Pixels outside the
// annulus [C_RADIUS - C_LINE/2, C_RADIUS + AMPLIFY + ...] are exactly 0 and skip the maths.
#define CIRCLE_TW 128
#define CIRCLE_TH 8
__global__ void __launch_bounds__(256, 5)
raster_circle_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int tiles_per_cta) {
    __shared__ uint32_t tile[CIRCLE_TH + 2][CIRCLE_TW + 2];
    const int stream = a.stream0 + blockIdx.z;
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    const int tx0 = blockIdx.x * CIRCLE_TW;
    const float cx = (float) (p.w / 2), cy = (float) (p.h / 2);
    // Static bounds of the annulus that can be lit, tightened per stream: a pixel is lit only if
    // d - C_RADIUS lies within [min(v) - C_LINE/2, max(v) + C_LINE/2] (circle/1.frag:72-80; v = AMPLIFY * texel over
    // the three fetched texels, 0 for out-of-range fetches), so the stream's texel range bounds its annulus.
    float reach = circle_reach(p);
    float inner = p.circle_radius - p.circle_line / 2.0f - 2.0f;
    if (a.texmm) {
        const uint32_t* mm = a.texmm + (size_t) stream * 2 * GLB_TEXMM_STRIDE;     // plane l, then plane r: {min, max} first
        const float f0 = from16(min(__ldg(mm + 0), __ldg(mm + GLB_TEXMM_STRIDE))) * p.circle_amplify;
        const float f1 = from16(max(__ldg(mm + 1), __ldg(mm + GLB_TEXMM_STRIDE + 1))) * p.circle_amplify;
        const float vlo = fminf(fminf(f0, f1), 0.0f), vhi = fmaxf(fmaxf(f0, f1), 0.0f);
        const float hl3 = fabsf(p.circle_line) / 2.0f + 3.0f;
        reach = fminf(reach, p.circle_radius + vhi + hl3);
        if (!p.circle_fill) inner = fmaxf(inner, p.circle_radius + vlo - hl3);
    }
    const float bx0 = (float) (tx0 - 1) - cx, bx1 = (float) (tx0 + CIRCLE_TW) - cx;
    const float nx = (bx0 > 0.0f) ? bx0 : ((bx1 < 0.0f) ? -bx1 : 0.0f);
    const float fxm = fmaxf(fabsf(bx0), fabsf(bx1));
    // 256 threads: 32 quads per row x 8 rows
    const int qx = threadIdx.x & 31, qy = threadIdx.x >> 5;
    const int x = tx0 + qx * 4;
    const CircleConsts cc = circle_consts(p);
    // whole CTA region (its 128 columns x tiles_per_cta*8 rows, + halo) outside the disc: bare zero-store loop
    {
        const int Y0 = blockIdx.y * tiles_per_cta * CIRCLE_TH, Y1 = min(p.h, Y0 + tiles_per_cta * CIRCLE_TH);
        const float cb0 = (float) (Y0 - 1) - cy, cb1 = (float) Y1 - cy;
        const float cny = (cb0 > 0.0f) ? cb0 : ((cb1 < 0.0f) ? -cb1 : 0.0f);
        if (nx * nx + cny * cny > reach * reach && (p.w & 3) == 0) {
            if (x < p.w) {
                const int stride = p.w >> 2;
                uint4* ptr = reinterpret_cast<uint4*>(fb) + (size_t) (Y0 + qy) * stride + (x >> 2);
                const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
                for (int y = Y0 + qy; y < Y1; y += CIRCLE_TH, ptr += (size_t) CIRCLE_TH * stride) __stcs(ptr, zero);
            }
            return;
        }
    }
    // a CTA walks `tiles_per_cta` vertically adjacent 128x8 tiles (a tile per CTA is too little work:
    // most tiles are outside the annulus and only store 4 KB of zeros)
    for (int it = 0; it < tiles_per_cta; ++it) {
        const int ty0 = (blockIdx.y * tiles_per_cta + it) * CIRCLE_TH;
        if (ty0 >= p.h) break;
        // distance range of the tile (+halo) from the centre
        const float by0 = (float) (ty0 - 1) - cy, by1 = (float) (ty0 + CIRCLE_TH) - cy;
        const float ny = (by0 > 0.0f) ? by0 : ((by1 < 0.0f) ? -by1 : 0.0f);
        const float fym = fmaxf(fabsf(by0), fabsf(by1));
        bool tile_dead = (nx * nx + ny * ny > reach * reach) || (inner > 0.0f && fxm * fxm + fym * fym < inner * inner);
        if (!tile_dead && a.ctile && a.texmm) {
            // the curve inside THIS tile's angular range: min / max over the texel buckets its cells can reference.  Every warp
            // reduces the same few buckets (no barrier; the outcome is CTA-uniform by construction)
            const int ti = (blockIdx.y * tiles_per_cta + it) * a.ctile_nx + blockIdx.x;
            const int4 tr = __ldg(a.ctile + ti);
            const int lane = threadIdx.x & 31, bs = t.n / GLB_CIRCLE_NB;
            const uint32_t* ml = a.texmm + (size_t) stream * 2 * GLB_TEXMM_STRIDE + 2;
            const uint32_t* mr = ml + GLB_TEXMM_STRIDE;
            uint32_t lo = 65535u, hi = 0u;
            bool any = __ldg(a.ctile_zero + ti) != 0;
            if (any) lo = 0u;                                   // an out-of-range reference reads 0
            if (tr.y >= tr.x) { any = true; for (int b = tr.x / bs + lane; b <= tr.y / bs; b += 32) { lo = min(lo, __ldg(ml + 2 * b)); hi = max(hi, __ldg(ml + 2 * b + 1)); } }
            if (tr.w >= tr.z) { any = true; for (int b = tr.z / bs + lane; b <= tr.w / bs; b += 32) { lo = min(lo, __ldg(mr + 2 * b)); hi = max(hi, __ldg(mr + 2 * b + 1)); } }
#pragma unroll
            for (int k = 16; k > 0; k >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, k)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, k)); }
            if (!any) tile_dead = true;                         // no cell of the tile (or its halo) can be lit
            else {
                if (hi < lo) hi = lo;
                const float g0 = from16(lo) * p.circle_amplify, g1 = from16(hi) * p.circle_amplify;
                const float tlo = fminf(g0, g1), thi = fmaxf(g0, g1);
                const float hl3 = fabsf(p.circle_line) / 2.0f + 3.0f;
                const float dnear = sqrtf(nx * nx + ny * ny) - p.circle_radius, dfar = sqrtf(fxm * fxm + fym * fym) - p.circle_radius;
                if (dnear > thi + hl3 || (!p.circle_fill && dfar < tlo - hl3)) tile_dead = true;
            }
        }
        if (!tile_dead) {
            // (batching the geometry loads of a thread's 5-6 cells ahead of the dependent texel fetches costs
            // registers and halves the resident warps; the live tiles are bound by instruction issue, not by the two
            // dependent L2 round trips.)
            if (a.geo) {
                // cached geometry: a cell is either outside the cache box (0) or a 16-byte entry with three
                // texel references + d; entries that cannot be lit carry e0 = -1.  No per-cell float culling,
                // no transcendental, constants hoisted (the kernel is instruction bound).
                const int4* __restrict__ geo = reinterpret_cast<const int4*>(a.geo);
                int ly = threadIdx.x / (CIRCLE_TW + 2), lx = threadIdx.x - ly * (CIRCLE_TW + 2);
                for (; ly < CIRCLE_TH + 2; ) {
                    const int bxi = tx0 + lx - 1 - a.gx0, byi = ty0 + ly - 1 - a.gy0;
                    uint32_t v = 0u;
                    if (bxi >= 0 && byi >= 0 && bxi < a.gw && byi < a.gh) {
                        const float dx = (float) (tx0 + lx - 1) - cx, dy = (float) (ty0 + ly - 1) - cy;
                        const float d2 = dx * dx + dy * dy;
                        if (d2 <= reach * reach && !(inner > 0.0f && d2 < inner * inner)) {   // per-stream annulus
                            const int4 e = __ldg(geo + (size_t) byi * a.gw + bxi);
                            CircleGeo g; g.dR = __int_as_float(e.x); g.e0 = e.y; g.e1 = e.z; g.e2 = e.w;
                            v = circle_stage1_c(cc, t.l, t.r, t.n, g);
                        }
                    }
                    tile[ly][lx] = v;
                    lx += 256 - (CIRCLE_TW + 2); ly += 1;               // advance by 256 cells: 256 = 130 + 126
                    if (lx >= CIRCLE_TW + 2) { lx -= CIRCLE_TW + 2; ly += 1; }
                }
            } else
            for (int i = threadIdx.x; i < (CIRCLE_TH + 2) * (CIRCLE_TW + 2); i += blockDim.x) {
                const int ly = i / (CIRCLE_TW + 2), lx = i - ly * (CIRCLE_TW + 2);
                const int gx = tx0 + lx - 1, gy = ty0 + ly - 1;
                uint32_t v = 0u;
                if (gx >= 0 && gy >= 0 && gx < p.w && gy < p.h) {
                    const float dx = (float) gx - cx, dy = (float) gy - cy;
                    const float d2 = dx * dx + dy * dy;
                    if (d2 <= reach * reach && !(inner > 0.0f && d2 < inner * inner)) v = circle_stage1(p, t, gx, gy);
                }
                tile[ly][lx] = v;
            }
            __syncthreads();
        }
        const int y = ty0 + qy;
        if (tile_dead) {
            if (x < p.w && y < p.h) { const uint32_t px[4] = { 0u, 0u, 0u, 0u }; store4(fb + (size_t) y * p.w, x, p.w, px); }
        } else if (y < p.h) {
            // live tile: a lane takes the pixels qx, qx + 32, qx + 64, qx + 96 of its row, so that the 7 tile reads per pixel
            // are CONSECUTIVE across the warp.  With 4 adjacent pixels per lane (one 128-bit store) every one of those reads
            // was a 4-way bank conflict, and the kernel is issue bound; four coalesced 4-byte stores per lane cost far less than that.
            uint32_t* row = fb + (size_t) y * p.w;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int cx = qx + 32 * k, gx = tx0 + cx;
                if (gx >= p.w) continue;
                const int lx = cx + 1, ly = qy + 1;
                // circle/2.frag's "- 1" taps at column 0 / row 0 read column 0 / row 0 (int(-0.5) = 0, see circle_px)
                const int lxm = (gx > 0) ? lx - 1 : lx, lym = (y > 0) ? ly - 1 : ly;
                const uint32_t own = tile[ly][lx];
                const uint32_t nb[6] = { tile[ly][lx + 1], tile[ly + 1][lx + 1], tile[ly + 1][lx],
                                         tile[ly][lxm], tile[lym][lxm], tile[lym][lx] };
                const uint32_t v = ((own | nb[0] | nb[1] | nb[2] | nb[3] | nb[4] | nb[5]) == 0u) ? 0u : circle_finish(p, own, nb);
                __stcs(row + gx, v);
            }
        }
        if (!tile_dead) __syncthreads();             // the tile is rewritten by the next iteration
    }
}
// styled twin (DESIGN 4.9): the same code reading its stream's style slot
__device__ __forceinline__ void circle_styled_body(const RasterArgs& a, int tiles_per_cta, const RasterStyles& sa) {
    __shared__ uint32_t tile[CIRCLE_TH + 2][CIRCLE_TW + 2];
    const int stream = a.stream0 + blockIdx.z;
    const glava_b200_params& p = stream_style<true>(sa, stream)->p;   // the cache is the slots' one
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    const int tx0 = blockIdx.x * CIRCLE_TW;
    const float cx = (float) (p.w / 2), cy = (float) (p.h / 2);
    // Static bounds of the annulus that can be lit, tightened per stream: a pixel is lit only if
    // d - C_RADIUS lies within [min(v) - C_LINE/2, max(v) + C_LINE/2] (circle/1.frag:72-80; v = AMPLIFY * texel over
    // the three fetched texels, 0 for out-of-range fetches), so the stream's texel range bounds its annulus.
    float reach = circle_reach(p);
    float inner = p.circle_radius - p.circle_line / 2.0f - 2.0f;
    if (a.texmm) {
        const uint32_t* mm = a.texmm + (size_t) stream * 2 * GLB_TEXMM_STRIDE;     // plane l, then plane r: {min, max} first
        const float f0 = from16(min(__ldg(mm + 0), __ldg(mm + GLB_TEXMM_STRIDE))) * p.circle_amplify;
        const float f1 = from16(max(__ldg(mm + 1), __ldg(mm + GLB_TEXMM_STRIDE + 1))) * p.circle_amplify;
        const float vlo = fminf(fminf(f0, f1), 0.0f), vhi = fmaxf(fmaxf(f0, f1), 0.0f);
        const float hl3 = fabsf(p.circle_line) / 2.0f + 3.0f;
        reach = fminf(reach, p.circle_radius + vhi + hl3);
        if (!p.circle_fill) inner = fmaxf(inner, p.circle_radius + vlo - hl3);
    }
    const float bx0 = (float) (tx0 - 1) - cx, bx1 = (float) (tx0 + CIRCLE_TW) - cx;
    const float nx = (bx0 > 0.0f) ? bx0 : ((bx1 < 0.0f) ? -bx1 : 0.0f);
    const float fxm = fmaxf(fabsf(bx0), fabsf(bx1));
    // 256 threads: 32 quads per row x 8 rows
    const int qx = threadIdx.x & 31, qy = threadIdx.x >> 5;
    const int x = tx0 + qx * 4;
    const CircleConsts cc = circle_consts(p);
    // whole CTA region (its 128 columns x tiles_per_cta*8 rows, + halo) outside the disc: bare zero-store loop
    {
        const int Y0 = blockIdx.y * tiles_per_cta * CIRCLE_TH, Y1 = min(p.h, Y0 + tiles_per_cta * CIRCLE_TH);
        const float cb0 = (float) (Y0 - 1) - cy, cb1 = (float) Y1 - cy;
        const float cny = (cb0 > 0.0f) ? cb0 : ((cb1 < 0.0f) ? -cb1 : 0.0f);
        if (nx * nx + cny * cny > reach * reach && (p.w & 3) == 0) {
            if (x < p.w) {
                const int stride = p.w >> 2;
                uint4* ptr = reinterpret_cast<uint4*>(fb) + (size_t) (Y0 + qy) * stride + (x >> 2);
                const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
                for (int y = Y0 + qy; y < Y1; y += CIRCLE_TH, ptr += (size_t) CIRCLE_TH * stride) __stcs(ptr, zero);
            }
            return;
        }
    }
    // a CTA walks `tiles_per_cta` vertically adjacent 128x8 tiles (a tile per CTA is too little work:
    // most tiles are outside the annulus and only store 4 KB of zeros)
    for (int it = 0; it < tiles_per_cta; ++it) {
        const int ty0 = (blockIdx.y * tiles_per_cta + it) * CIRCLE_TH;
        if (ty0 >= p.h) break;
        // distance range of the tile (+halo) from the centre
        const float by0 = (float) (ty0 - 1) - cy, by1 = (float) (ty0 + CIRCLE_TH) - cy;
        const float ny = (by0 > 0.0f) ? by0 : ((by1 < 0.0f) ? -by1 : 0.0f);
        const float fym = fmaxf(fabsf(by0), fabsf(by1));
        bool tile_dead = (nx * nx + ny * ny > reach * reach) || (inner > 0.0f && fxm * fxm + fym * fym < inner * inner);
        if (!tile_dead && a.ctile && a.texmm) {
            // the curve inside THIS tile's angular range: min / max over the texel buckets its cells can reference.  Every warp
            // reduces the same few buckets (no barrier; the outcome is CTA-uniform by construction)
            const int ti = (blockIdx.y * tiles_per_cta + it) * a.ctile_nx + blockIdx.x;
            const int4 tr = __ldg(a.ctile + ti);
            const int lane = threadIdx.x & 31, bs = t.n / GLB_CIRCLE_NB;
            const uint32_t* ml = a.texmm + (size_t) stream * 2 * GLB_TEXMM_STRIDE + 2;
            const uint32_t* mr = ml + GLB_TEXMM_STRIDE;
            uint32_t lo = 65535u, hi = 0u;
            bool any = __ldg(a.ctile_zero + ti) != 0;
            if (any) lo = 0u;                                   // an out-of-range reference reads 0
            if (tr.y >= tr.x) { any = true; for (int b = tr.x / bs + lane; b <= tr.y / bs; b += 32) { lo = min(lo, __ldg(ml + 2 * b)); hi = max(hi, __ldg(ml + 2 * b + 1)); } }
            if (tr.w >= tr.z) { any = true; for (int b = tr.z / bs + lane; b <= tr.w / bs; b += 32) { lo = min(lo, __ldg(mr + 2 * b)); hi = max(hi, __ldg(mr + 2 * b + 1)); } }
#pragma unroll
            for (int k = 16; k > 0; k >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, k)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, k)); }
            if (!any) tile_dead = true;                         // no cell of the tile (or its halo) can be lit
            else {
                if (hi < lo) hi = lo;
                const float g0 = from16(lo) * p.circle_amplify, g1 = from16(hi) * p.circle_amplify;
                const float tlo = fminf(g0, g1), thi = fmaxf(g0, g1);
                const float hl3 = fabsf(p.circle_line) / 2.0f + 3.0f;
                const float dnear = sqrtf(nx * nx + ny * ny) - p.circle_radius, dfar = sqrtf(fxm * fxm + fym * fym) - p.circle_radius;
                if (dnear > thi + hl3 || (!p.circle_fill && dfar < tlo - hl3)) tile_dead = true;
            }
        }
        if (!tile_dead) {
            // (batching the geometry loads of a thread's 5-6 cells ahead of the dependent texel fetches costs
            // registers and halves the resident warps; the live tiles are bound by instruction issue, not by the two
            // dependent L2 round trips.)
            if (a.geo) {
                // cached geometry: a cell is either outside the cache box (0) or a 16-byte entry with three
                // texel references + d; entries that cannot be lit carry e0 = -1.  No per-cell float culling,
                // no transcendental, constants hoisted (the kernel is instruction bound).
                const int4* __restrict__ geo = reinterpret_cast<const int4*>(a.geo);
                int ly = threadIdx.x / (CIRCLE_TW + 2), lx = threadIdx.x - ly * (CIRCLE_TW + 2);
                for (; ly < CIRCLE_TH + 2; ) {
                    const int bxi = tx0 + lx - 1 - a.gx0, byi = ty0 + ly - 1 - a.gy0;
                    uint32_t v = 0u;
                    if (bxi >= 0 && byi >= 0 && bxi < a.gw && byi < a.gh) {
                        const float dx = (float) (tx0 + lx - 1) - cx, dy = (float) (ty0 + ly - 1) - cy;
                        const float d2 = dx * dx + dy * dy;
                        if (d2 <= reach * reach && !(inner > 0.0f && d2 < inner * inner)) {   // per-stream annulus
                            const int4 e = __ldg(geo + (size_t) byi * a.gw + bxi);
                            CircleGeo g; g.dR = __int_as_float(e.x); g.e0 = e.y; g.e1 = e.z; g.e2 = e.w;
                            v = circle_stage1_c(cc, t.l, t.r, t.n, g);
                        }
                    }
                    tile[ly][lx] = v;
                    lx += 256 - (CIRCLE_TW + 2); ly += 1;               // advance by 256 cells: 256 = 130 + 126
                    if (lx >= CIRCLE_TW + 2) { lx -= CIRCLE_TW + 2; ly += 1; }
                }
            } else
            for (int i = threadIdx.x; i < (CIRCLE_TH + 2) * (CIRCLE_TW + 2); i += blockDim.x) {
                const int ly = i / (CIRCLE_TW + 2), lx = i - ly * (CIRCLE_TW + 2);
                const int gx = tx0 + lx - 1, gy = ty0 + ly - 1;
                uint32_t v = 0u;
                if (gx >= 0 && gy >= 0 && gx < p.w && gy < p.h) {
                    const float dx = (float) gx - cx, dy = (float) gy - cy;
                    const float d2 = dx * dx + dy * dy;
                    if (d2 <= reach * reach && !(inner > 0.0f && d2 < inner * inner)) v = circle_stage1(p, t, gx, gy);
                }
                tile[ly][lx] = v;
            }
            __syncthreads();
        }
        const int y = ty0 + qy;
        if (tile_dead) {
            if (x < p.w && y < p.h) { const uint32_t px[4] = { 0u, 0u, 0u, 0u }; store4(fb + (size_t) y * p.w, x, p.w, px); }
        } else if (y < p.h) {
            // live tile: a lane takes the pixels qx, qx + 32, qx + 64, qx + 96 of its row, so that the 7 tile reads per pixel
            // are CONSECUTIVE across the warp.  With 4 adjacent pixels per lane (one 128-bit store) every one of those reads
            // was a 4-way bank conflict, and the kernel is issue bound; four coalesced 4-byte stores per lane cost far less than that.
            uint32_t* row = fb + (size_t) y * p.w;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int cx = qx + 32 * k, gx = tx0 + cx;
                if (gx >= p.w) continue;
                const int lx = cx + 1, ly = qy + 1;
                // circle/2.frag's "- 1" taps at column 0 / row 0 read column 0 / row 0 (int(-0.5) = 0, see circle_px)
                const int lxm = (gx > 0) ? lx - 1 : lx, lym = (y > 0) ? ly - 1 : ly;
                const uint32_t own = tile[ly][lx];
                const uint32_t nb[6] = { tile[ly][lx + 1], tile[ly + 1][lx + 1], tile[ly + 1][lx],
                                         tile[ly][lxm], tile[lym][lxm], tile[lym][lx] };
                const uint32_t v = ((own | nb[0] | nb[1] | nb[2] | nb[3] | nb[4] | nb[5]) == 0u) ? 0u : circle_finish(p, own, nb);
                __stcs(row + gx, v);
            }
        }
        if (!tile_dead) __syncthreads();             // the tile is rewritten by the next iteration
    }
}
__global__ void __launch_bounds__(256, 5)
raster_circle_styled_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params, int tiles_per_cta,
                            const __grid_constant__ RasterStyles sa) {
    circle_styled_body(a, tiles_per_cta, sa);
}
// radial: per-pixel polar maths (radial/1.frag + premultiply) with disc culling; same arithmetic as
// raster_generic_kernel but without the module switch (no spills).
template <bool STYLED>
__device__ __forceinline__ void radial_body(const RasterArgs& a, const glava_b200_params& pk, int rows_per_cta, const RasterStyles& sa) {
    const int stream = a.stream0 + blockIdx.z;
    const glava_b200_params& p = style_params_of<STYLED>(stream_style<STYLED>(sa, stream), pk);
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    const AudioTex t = make_tex(p, a.tex, stream);
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    const float reach = radial_reach(p), r2 = reach * reach;
    const float cx = (float) (p.w / 2) - p.radial_off_x, cy = (float) (p.h / 2) - p.radial_off_y;
    const float dxa = (float) x - cx, dxb = (float) (x + 3) - cx;
    float dxm = ((dxa > 0.0f) ? dxa : ((dxb < 0.0f) ? -dxb : 0.0f)) - 1.0f;     // span distance from cx, 1 px slack
    if (dxm < 0.0f) dxm = 0.0f;
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    for (int y = y0; y < y1; ++y) {
        uint32_t px[4] = { 0u, 0u, 0u, 0u };
        float dy = fabsf((float) y - cy) - 1.0f;
        if (dy < 0.0f) dy = 0.0f;
        if (dxm * dxm + dy * dy <= r2) {
#pragma unroll
            for (int k = 0; k < 4; ++k) if (x + k < p.w) px[k] = radial_px(p, t, x + k, y);
        }
        store4(fb + (size_t) y * p.w, x, p.w, px);
    }
}
GLB_STYLED_PAIR(radial_body, __launch_bounds__(128), raster_radial_kernel, raster_radial_styled_kernel)

// per-plane {min, max} of the R16 texture the module samples (circle: bounds the stream's annulus), followed by the
// {min, max} of GLB_CIRCLE_NB buckets of n / GLB_CIRCLE_NB consecutive texels (bounds a TILE's annulus: a tile's cells
// reference a known range of texels, see circle_tile_kernel)
__global__ void __launch_bounds__(256)
texmm_kernel(const uint16_t* __restrict__ tex, int n, uint32_t* __restrict__ out) {
    __shared__ uint32_t smin[8], smax[8];
    const uint16_t* t = tex + (size_t) blockIdx.x * n;
    uint32_t* o = out + (size_t) blockIdx.x * GLB_TEXMM_STRIDE;
    const int per = n / 256;                                  // n >= 256: thread t covers [t * per, (t + 1) * per), two threads per bucket
    uint32_t lo = 65535u, hi = 0u;
    for (int i = 0; i < per; ++i) { const uint32_t v = t[threadIdx.x * per + i]; lo = min(lo, v); hi = max(hi, v); }
    {
        const uint32_t blo = min(lo, __shfl_xor_sync(0xffffffffu, lo, 1)), bhi = max(hi, __shfl_xor_sync(0xffffffffu, hi, 1));
        if ((threadIdx.x & 1) == 0) { o[2 + threadIdx.x] = blo; o[3 + threadIdx.x] = bhi; }      // bucket threadIdx.x / 2
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, k)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, k)); }
    if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = lo; smax[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) { lo = min(lo, smin[w]); hi = max(hi, smax[w]); }
        o[0] = lo; o[1] = hi;
    }
}
int launch_texmm(const glava_b200_params& p, const uint16_t* d_tex, uint32_t* d_out, int planes, void* stream) {
    texmm_kernel<<<planes, 256, 0, (cudaStream_t) stream>>>(d_tex, p.n, d_out);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "texmm kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// ---- polar geometry cache (raster_plan.h polar_geo_box) -----------------------------------------------------------------
__global__ void polar_geo_kernel(int4* __restrict__ geo, int gx0, int gy0, int gw, int gh, const __grid_constant__ glava_b200_params p) {
    const int bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y;
    if (bx >= gw || by >= gh) return;
    const int x = gx0 + bx, y = gy0 + by;
    int4 out;
    if (p.module == GLAVA_B200_MOD_RADIAL) {
        RadialGeo g = { 0u, 0u, 0.0f, -1, 0u };
        if (x < p.w) g = radial_geometry(p, x, y);
        out = make_int4((int) g.lit, (int) g.unlit, __float_as_int(g.dR), g.bar);
        // compact levels read by raster_radial_geo_kernel: 1-byte class code per pixel
        //   0        pixel is always 0
        //   1..254   plain bar pixel (unlit value 0): 1 + side * nk + k, its {lit, dR} in the 8-byte level
        //   255      anything else (ring zone, bar id that does not fit): full 16-byte entry
        const size_t npx = (size_t) gw * gh, at = (size_t) by * gw + bx;
        int2* bar8 = reinterpret_cast<int2*>(geo + npx);
        unsigned char* code = reinterpret_cast<unsigned char*>(bar8 + npx);
        const int nk = p.radial_nbars / 2 + 2;
        int c;
        if (g.bar < 0) c = (g.unlit == 0u) ? 0 : 255;
        else {
            const int id = 1 + (g.bar >> 16) * nk + (g.bar & 0xffff);
            c = (g.unlit == 0u && (g.bar & 0xffff) < nk && id <= 254) ? id : 255;
        }
        bar8[at] = make_int2((int) g.lit, __float_as_int(g.dR));
        code[at] = (unsigned char) c;
    } else {
        CircleGeo g = circle_geometry(p, x, y);          // handles x >= w
        out = make_int4(__float_as_int(g.dR), g.e0, g.e1, g.e2);
    }
    geo[(size_t) by * gw + bx] = out;
}
int launch_polar_geo(const glava_b200_params& p, void* d_geo, const int box[4], void* stream) {
    dim3 grid((box[2] + 127) / 128, box[3]);
    polar_geo_kernel<<<grid, 128, 0, (cudaStream_t) stream>>>(reinterpret_cast<int4*>(d_geo), box[0], box[1], box[2], box[3], p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "polar geometry kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// circle: which texels can the cells of a 128 x 8 tile (+ its 1-pixel halo, read by stage 2) reference?  Audio-independent,
// so it is reduced once from the finished cache; per frame and stream the buckets of texmm_kernel then bound the curve
// INSIDE the tile's angular range, and a tile the curve cannot touch costs 4 KB of zero stores instead of 1300 cell
// evaluations (the per-stream annulus alone keeps every tile between the base circle and the tallest peak alive).
size_t circle_tile_bytes(const glava_b200_params& p, int* ntx, int* nty) {
    *ntx = (p.w + CIRCLE_TW - 1) / CIRCLE_TW; *nty = (p.h + CIRCLE_TH - 1) / CIRCLE_TH;
    return (size_t) *ntx * *nty * (sizeof(int4) + sizeof(int));
}
__global__ void circle_tile_init_kernel(int4* tiles, int* zero, int count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) { tiles[i] = make_int4(0x7fffffff, -1, 0x7fffffff, -1); zero[i] = 0; }
}
__global__ void circle_tile_kernel(const int4* __restrict__ geo, int gx0, int gy0, int gw, int gh, int4* tiles, int* zero, int ntx, int nty) {
    const int bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y;
    if (bx >= gw || by >= gh) return;
    const int4 e = geo[(size_t) by * gw + bx];
    if (e.y < 0) return;                                                   // the cell cannot be lit: it references nothing
    int lo[2] = { 0x7fffffff, 0x7fffffff }, hi[2] = { -1, -1 }, z = 0;
    const int refs[3] = { e.y, e.z, e.w };
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int ch = (refs[k] >> 30) & 1, i = refs[k] & 0x3fffffff;
        if (i == 0x3fffffff) z = 1; else { lo[ch] = min(lo[ch], i); hi[ch] = max(hi[ch], i); }
    }
    const int x = gx0 + bx, y = gy0 + by;
    int seen[4] = { -1, -1, -1, -1 }, ns = 0;
    for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {                                 // every tile whose halo contains this cell
            const int tx = (x + dx) / CIRCLE_TW, ty = (y + dy) / CIRCLE_TH;
            if (x + dx < 0 || y + dy < 0 || tx >= ntx || ty >= nty) continue;
            const int ti = ty * ntx + tx;
            bool dup = false;
            for (int q = 0; q < ns; ++q) dup |= seen[q] == ti;
            if (dup) continue;
            if (ns < 4) seen[ns++] = ti;
            int* t = reinterpret_cast<int*>(tiles + ti);
            if (hi[0] >= 0) { atomicMin(t + 0, lo[0]); atomicMax(t + 1, hi[0]); }
            if (hi[1] >= 0) { atomicMin(t + 2, lo[1]); atomicMax(t + 3, hi[1]); }
            if (z) atomicOr(zero + ti, 1);
        }
}
int launch_circle_tiles(const glava_b200_params& p, const void* d_geo, const int box[4], void* d_tiles, void* stream) {
    int ntx, nty;
    circle_tile_bytes(p, &ntx, &nty);
    int4* tiles = reinterpret_cast<int4*>(d_tiles);
    int* zero = reinterpret_cast<int*>(tiles + (size_t) ntx * nty);
    cudaStream_t st = (cudaStream_t) stream;
    circle_tile_init_kernel<<<(ntx * nty + 255) / 256, 256, 0, st>>>(tiles, zero, ntx * nty);
    dim3 grid((box[2] + 127) / 128, box[3]);
    circle_tile_kernel<<<grid, 128, 0, st>>>(reinterpret_cast<const int4*>(d_geo), box[0], box[1], box[2], box[3], tiles, zero, ntx, nty);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "circle tile kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// radial from the geometry cache: per pixel one 16-byte load, one compare against the bar's height
// (160 heights per stream, in shared memory), one select.
// `geo_cache` is a.geo (plain) or the slot's cache (styled).  `a` is taken by value: taken by reference, the plain kernel
// compiles to other machine code (DESIGN 4.9).
__device__ __forceinline__ void radial_geo_body(const RasterArgs a, const glava_b200_params& p, const void* geo_cache,
                                                int rows_per_cta) {
    __shared__ float vflat[RADIAL_MAX_BARS + 4];        // bar heights, index side * nk + k (== class code - 1)
    __shared__ float vmax_s;                             // tallest bar of this stream
    const int stream = a.stream0 + blockIdx.z;
    const AudioTex t = make_tex(p, a.tex, stream);
    const int nk = p.radial_nbars / 2 + 2;               // k = int(|idx| / section) <= NBARS / 2 (+1 for rounding)
    const int y0 = blockIdx.y * rows_per_cta, y1 = min(p.h, y0 + rows_per_cta);
    const bool band_live = (y1 > a.gy0) && (y0 < a.gy0 + a.gh);
    if (band_live) {
        for (int i = threadIdx.x; i < 2 * nk; i += blockDim.x) {
            const int side = i / nk, k = i - side * nk;
            vflat[i] = radial_bar_value(p, t, (side << 16) | k);
        }
        __syncthreads();
        if (threadIdx.x < 32) {                          // tallest bar: nothing beyond C_RADIUS + vmax can be lit
            float m = 0.0f;
            for (int i = threadIdx.x; i < 2 * nk; i += 32) m = fmaxf(m, vflat[i]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            if (threadIdx.x == 0) vmax_s = m;
        }
        __syncthreads();
    }
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= p.w) return;
    // per-stream reach: a bar pixel is lit only if d - C_RADIUS <= v <= vmax; beyond that (and beyond the ring) the
    // frame is 0 for THIS stream, so those quads skip the geometry loads (typical spectra reach a third of AMPLIFY)
    const float rcull = band_live ? p.radial_radius + fmaxf(fmaxf(vmax_s, 0.0f), fabsf(p.radial_line)) + 2.0f : 0.0f;
    const float ccx = (float) (p.w / 2) - p.radial_off_x, ccy = (float) (p.h / 2) - p.radial_off_y;
    float qdx; {
        const float dxa = (float) x - ccx, dxb = (float) (x + 4) - ccx;          // pixel centres are at +0.5: [x, x+4) covers them
        qdx = (dxa > 0.0f) ? dxa : ((dxb < 0.0f) ? -dxb : 0.0f);
        qdx = fmaxf(qdx - 1.0f, 0.0f);
    }
    uint32_t* fb = reinterpret_cast<uint32_t*>(a.fb) + (size_t) (stream % a.slots) * p.w * p.h;
    const size_t npx = (size_t) a.gw * a.gh;
    const int4* __restrict__ geo = reinterpret_cast<const int4*>(geo_cache);                // full entries
    const int2* __restrict__ bar8 = reinterpret_cast<const int2*>(geo + npx);               // {lit, dR}
    const unsigned char* __restrict__ code = reinterpret_cast<const unsigned char*>(bar8 + npx);
    const int bxi = x - a.gx0;
    const bool col_live = bxi >= 0 && bxi < a.gw;        // gx0, gw multiples of 4: the quad is inside or outside as a whole
    // One row per trip on purpose: batching the loads of 4 rows (more memory-level parallelism per warp)
    // raises the register count enough to halve the resident warps, and even the pure zero-store rows
    // outside the box need the occupancy.
    for (int y = y0; y < y1; ++y) {
        uint32_t px[4] = { 0u, 0u, 0u, 0u };
        const int byi = y - a.gy0;
        const float qdy = fmaxf(fabsf((float) y + 0.5f - ccy) - 1.0f, 0.0f);
        if (col_live && byi >= 0 && byi < a.gh && qdx * qdx + qdy * qdy <= rcull * rcull) {
            const size_t at = (size_t) byi * a.gw + bxi;
            // codes and {lit, dR} are fetched together (independent addresses): one L2 round trip per
            // row instead of two dependent ones — the row loop is latency x occupancy bound
            const uint32_t codes = __ldg(reinterpret_cast<const uint32_t*>(code + at));       // 4 pixels
            const int4 e01 = __ldg(reinterpret_cast<const int4*>(bar8 + at));                 // pixels 0, 1
            const int4 e23 = __ldg(reinterpret_cast<const int4*>(bar8 + at) + 1);             // pixels 2, 3
            if (codes != 0u) {
                const int2 e8[4] = { make_int2(e01.x, e01.y), make_int2(e01.z, e01.w), make_int2(e23.x, e23.y), make_int2(e23.z, e23.w) };
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint32_t c = (codes >> (8 * k)) & 255u;
                    if (c == 0u) continue;
                    if (c != 255u) {
                        const int2 e = e8[k];
                        if (__int_as_float(e.y) <= vflat[c - 1u]) px[k] = (uint32_t) e.x;
                    } else {
                        const int4 e = __ldg(geo + at + k);            // {lit, unlit, dR, bar}
                        uint32_t v = (uint32_t) e.y;
                        if (e.w >= 0) {
                            const int kk = e.w & 0xffff;
                            const float vb = kk < nk ? vflat[(e.w >> 16) * nk + kk] : radial_bar_value(p, t, e.w);
                            if (__int_as_float(e.z) <= vb) v = (uint32_t) e.x;
                        }
                        px[k] = v;
                    }
                }
            }
        }
        store4(fb + (size_t) y * p.w, x, p.w, px);
    }
}
__global__ void __launch_bounds__(128)
raster_radial_geo_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params p, int rows_per_cta) {
    radial_geo_body(a, p, a.geo, rows_per_cta);
}
__global__ void __launch_bounds__(128)
raster_radial_geo_styled_kernel(const __grid_constant__ RasterArgs a, const __grid_constant__ glava_b200_params, int rows_per_cta,
                                const __grid_constant__ RasterStyles sa) {
    const StyleSlot* const sty = stream_style<true>(sa, a.stream0 + blockIdx.z);
    radial_geo_body(a, sty->p, sty->geo, rows_per_cta);      // the slot's colours' cache
}

// One launch of a plain kernel or of its styled twin (the style slots as the last parameter, room for a slot's copy as
// dynamic shared memory)
template <bool S>
static void launch_one(void (*plain)(RasterArgs, glava_b200_params, int), void (*styled)(RasterArgs, glava_b200_params, int, RasterStyles),
                       dim3 grid, int threads, cudaStream_t st, const RasterArgs& b, const glava_b200_params& p, const RasterStyles& sa, int n) {
    if constexpr (S) styled<<<grid, threads, sizeof(StyleSlot), st>>>(b, p, n, sa);
    else plain<<<grid, threads, 0, st>>>(b, p, n);
}
template <bool S>
static void launch_one(void (*plain)(RasterArgs, glava_b200_params), void (*styled)(RasterArgs, glava_b200_params, RasterStyles),
                       dim3 grid, int threads, cudaStream_t st, const RasterArgs& b, const glava_b200_params& p, const RasterStyles& sa) {
    if constexpr (S) styled<<<grid, threads, sizeof(StyleSlot), st>>>(b, p, sa);
    else plain<<<grid, threads, 0, st>>>(b, p);
}
// The kernels of one chunk of streams, plain (S = false) or styled
template <bool S>
static void launch_chunk(const glava_b200_params& p, const RasterPlan& pl, const RasterArgs& b, const RasterStyles& sa, int nz, cudaStream_t st) {
    const int quads = (p.w + 3) / 4;
    const dim3 grid((quads + pl.bx - 1) / pl.bx, (p.h + pl.rows - 1) / pl.rows, nz);
    const dim3 tg((p.w + 127) / 128, nz);                  // column_table_kernel: a thread per column
    const int r = pl.rows;
    switch (pl.kernel) {
    case RasterKernel::GENERIC: launch_one<S>(raster_generic_kernel, raster_generic_styled_kernel, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::BARS: launch_one<S>(raster_bars_kernel, raster_bars_styled_kernel, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::GRAPH: launch_one<S>(raster_graph_kernel<false, 1>, raster_graph_styled_kernel<false, 1>, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::GRAPH_TAB4:
        launch_one<S>(column_table_kernel<false>, column_table_styled_kernel<false>, tg, 128, st, b, p, sa);
        launch_one<S>(raster_graph_kernel<true, 4>, raster_graph_styled_kernel<true, 4>, grid, pl.bx, st, b, p, sa, r);
        break;
    case RasterKernel::GRAPH_TAB5:
        launch_one<S>(column_table_kernel<false>, column_table_styled_kernel<false>, tg, 128, st, b, p, sa);
        launch_one<S>(raster_graph_kernel<true, 5>, raster_graph_styled_kernel<true, 5>, grid, pl.bx, st, b, p, sa, r);
        break;
    case RasterKernel::WAVE: launch_one<S>(raster_wave_kernel<false, 1>, raster_wave_styled_kernel<false, 1>, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::WAVE_TAB4:
        launch_one<S>(column_table_kernel<true>, column_table_styled_kernel<true>, tg, 128, st, b, p, sa);
        launch_one<S>(raster_wave_kernel<true, 4>, raster_wave_styled_kernel<true, 4>, grid, pl.bx, st, b, p, sa, r);
        break;
    case RasterKernel::WAVE_TAB5:
        launch_one<S>(column_table_kernel<true>, column_table_styled_kernel<true>, tg, 128, st, b, p, sa);
        launch_one<S>(raster_wave_kernel<true, 5>, raster_wave_styled_kernel<true, 5>, grid, pl.bx, st, b, p, sa, r);
        break;
    case RasterKernel::RADIAL: launch_one<S>(raster_radial_kernel, raster_radial_styled_kernel, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::RADIAL_GEO: launch_one<S>(raster_radial_geo_kernel, raster_radial_geo_styled_kernel, grid, pl.bx, st, b, p, sa, r); break;
    case RasterKernel::CIRCLE: {
        const int ntile_y = (p.h + CIRCLE_TH - 1) / CIRCLE_TH;
        const dim3 cgrid((p.w + CIRCLE_TW - 1) / CIRCLE_TW, (ntile_y + pl.circle_tiles - 1) / pl.circle_tiles, nz);
        launch_one<S>(raster_circle_kernel, raster_circle_styled_kernel, cgrid, pl.bx, st, b, p, sa, pl.circle_tiles);
        break;
    }
    }
}

int launch_raster(const glava_b200_params& p, const RasterPlan& pl, const RasterArgs& a, void* stream) {
    cudaStream_t st = (cudaStream_t) stream;
    const RasterStyles sa = pl.styled ? static_cast<const RasterPass&>(a).styles : RasterStyles{};
    if (pl.mark_key && !a.marks) return fail(GLAVA_B200_EINVAL, "raster launch: no dirty-row marks for the bars / graph / wave kernel");
    if (pl.styled && (!sa.style_of || !sa.styles)) return fail(GLAVA_B200_EINVAL, "raster launch: no style slots for the styled kernels");
    for (int s0 = 0; s0 < a.batch; s0 += pl.chunk) {
        RasterArgs b = a; b.stream0 = a.stream0 + s0;
        const int nz = a.batch - s0 < pl.chunk ? a.batch - s0 : pl.chunk;
        if (pl.styled) launch_chunk<true>(p, pl, b, sa, nz, st);
        else launch_chunk<false>(p, pl, b, sa, nz, st);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "raster kernel launch: %s", cudaGetErrorString(e));
    }
    return 0;
}

}  // namespace glb
