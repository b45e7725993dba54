// internal.h — shared declarations of libglava_b200 (host side + kernel launchers).
#ifndef GLAVA_B200_INTERNAL_H
#define GLAVA_B200_INTERNAL_H

#include "../../include/glava_b200.h"

#include <cstddef>
#include <cstdint>

namespace glb {

// error reporting: stores the message, calls the abort hook (glava.h:17 analogue), returns `code`
int  fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
void clear_error();
bool has_error();

// config.cpp
void fill_defaults(glava_b200_params* p, int module);
int  module_from_name(const char* name);
const char* module_name(int id);
bool parse_hex_color(const char* s, float out[4], bool literal_rounding);
bool parse_hex_components(const char* s, float* out[4]);
int  load_config(glava_b200_params* out, const char* const* paths, const char* entry,
                 const char* const* requests, const char* force_module, const char* const* binds);
int  validate_params(const glava_b200_params* p);
int  style_apply(const glava_b200_params& base, const glava_b200_stream_style& s, glava_b200_params* out);   // capi.cu

#define GLB_MAX_AVG_FRAMES 16

#ifndef GLB_TAPENTRY_DEFINED
#define GLB_TAPENTRY_DEFINED
struct alignas(8) TapEntry { int idx; float w; };   // one tap of the K5 smoothing sum: texel index, weight
#endif

// ---- views handed to the kernels (all pointers are DEVICE pointers) ---------------------------
// "channel plane" c = stream * 2 + ch (ch 0 = left, 1 = right); every per-channel array is
// [batch*2][...] so one CTA of the spectrum kernel owns one contiguous plane.
struct SpectrumArgs {
    const float*  pcm_l;        // [batch][n]   ring contents, oldest first (glava.c:528-537 lb)
    const float*  pcm_r;        // [batch][n]
    const double* window;       // [n]          render.c:660,794 window LUT (double, as the macro evaluates)
    const float*  twiddle;      // [n/2][2]     exp(-2*pi*i*k/(n/2)) as (re, im)
    float*    spec;             // [batch*2][n] pipeline-A result, or raw transform_fft output (accel)
    float*    applied;          // [batch*2][n] transform_gravity state (A), render.c:725
    float*    ring_f;           // [batch*2][F][n] transform_average ring (A), slot = update index % F
    uint16_t* gr_store;         // [batch*2][n] (B) render.c:2197
    uint16_t* ring_u;           // [batch*2][F][n] (B) gr->out[], render.c:2232
    uint16_t* tex;              // [batch*2][n] R16 texture the module samples
    uint16_t* av_out;           // non-null: export the pre-smoothing texture here and skip K5 (k5_planes_kernel follows)
    const int* need;            // lazy K5: texel indices to evaluate, [2][need_count] (-1 = unused), nullptr = all n
    int       need_count;
    // precomputed K5 taps for the need-list (weights and indices do not depend on the audio):
    const TapEntry* tap_tab;    // [2][tap_max][need_count], tap-major so a warp's loads coalesce; nullptr = evaluate directly
    const int*   tap_cnt;       // [2][need_count]
    const float* tap_wsum;      // [2][need_count]  sum of the weights in loop order
    int       tap_max;
    int       tap_ku;           // table entries a thread keeps in flight (8, 4 or 2)
    int       epi_n;            // lazy K5: number of leading bins whose gravity/average state can reach a sampled texel (0 = all)
    // the same taps as one blob per channel, small enough to live in shared memory (loaded by the TMA engine while the
    // FFT runs): [float w[csr_total]] [uint16 idx[csr_total]] [int off[need_count + 1]], texel-major ("CSR"); nullptr = unused
    const unsigned char* csr;   // [2][csr_bytes]
    int       csr_bytes;        // bytes per channel (multiple of 16)
    int       csr_idx_off, csr_off_off;   // byte offsets of idx[] and off[] inside a blob
    int       skip_tex;         // 1: produce `spec` only (transform_smooth / keyframe lerp / upload / K5 follow as kernels)
    int       batch;
    unsigned long long update;  // number of modified updates before this one (ring cursor)
    // per-stream `modified` (glava.c:528-537 decides per renderer, i.e. per stream): nullptr = every stream is modified and
    // shares the cursor `update % F`; else one word per stream, bit 31 = this stream has new audio, low 16 bits = its own
    // ring cursor (modified updates of THAT stream so far, mod F).  An unmodified stream's state is left alone and its
    // texture is carried from `tex_prev` (the half of the double buffer the previous raster read) into `tex`.
    int variant_oop, variant_t; // kernel variant: out-of-place passes, threads per CTA (0 = the size's default)
    int fft_only;               // 1: stop after transform_fft — `spec` (the leading epi_n bins) is all this launch produces; gravity /
                                // average run as epilogue_b_kernel, K5 as k5_need_smem_kernel / k5_need_kernel (launch_spectrum_update)
    int av_t_len;               // > 0: av_out receives only the leading av_t_len bins (need-list K5 as its own kernel downstream)
    const uint32_t* umask;      // [batch]
    const uint16_t* tex_prev;   // [batch*2][n]
    double    avg_w_a[GLB_MAX_AVG_FRAMES];   // pipeline A weights, oldest first (render.c:661,766)
    float     avg_w_b[GLB_MAX_AVG_FRAMES];   // pipeline B weights, newest first (average_pass.frag:41)
    int       avg_b_windowed;                // average_pass.frag:27-29,38-42
};

struct RasterArgs {
    const uint16_t* tex;        // [batch*2][n]
    uint8_t*  fb;               // [slots][h][w][4]
    const void* rowtab;         // module row table (bars: [h] {fill, outline} RGBA8 pairs), may be null
    int       batch, slots, stream0;
    // polar modules: per-renderer cache of the audio-independent per-pixel geometry (RadialGeo /
    // CircleGeo, 16 bytes each) over the bounding box of the disc that can be non-zero; may be null
    const void* geo;
    int       gx0, gy0, gw, gh;  // box origin and size in pixels (gx0, gw multiples of 4)
    const uint32_t* texmm;       // circle: per plane of `tex` {min, max} followed by GLB_CIRCLE_NB bucket {min, max} pairs (may be null)
    // circle: per 128 x 8 tile (+ 1-pixel halo) the range of texel indices its cells reference, {lo_l, hi_l, lo_r, hi_r}
    // (lo > hi: none), and whether any reference is out of range (reads 0); audio-independent, built with the cache
    const int4* ctile; const int* ctile_zero; int ctile_nx;
    // graph / wave: per-stream column table [batch][GLB_COLTAB_PLANES][w] floats, scratch that launch_raster fills on the
    // raster stream right before the module kernel (graph: plane 0 = column height; wave: WaveCol's five fields); may be null
    float* coltab;
    // bars / graph / wave: dirty-row marks (raster_core.h dirty_pack), [slots][h][(w + 127) / 128] words, a band's word at
    // its first row.  marks_valid = 0: the words do not describe the framebuffer (another kernel or band height wrote it
    // last); the kernel then stores every zero row and writes fresh marks.  run_update sets it (raster_plan.h raster_marks_valid).
    uint32_t* marks;
    int       marks_valid;
};
// Stream styles (DESIGN 4.9): the style slot of every stream [batch] and the slots' records [style slots] (slot 0: the
// renderer's own look).  A parameter of the styled kernel instantiations only, after the others: RasterArgs keeps its
// layout, so the plain kernels keep their parameter offsets and machine code.
struct RasterStyles {
    const int* style_of;
    const struct StyleSlot* styles;
};
// What capi.cu hands launch_raster: the kernels' RasterArgs and, for the styled instantiations, the style slots
struct RasterPass : RasterArgs {
    RasterStyles styles;
};
// One style slot as the styled raster kernels see it: the raster view of the styled parameters and the slot's tables
// (bars / graph row table, radial geometry cache; circle: the one cache).  Copied whole into shared memory by every CTA.
struct alignas(16) StyleSlot {
    glava_b200_params p;
    const void* rowtab;
    const void* geo;
};
#define GLB_COLTAB_PLANES 5
#define GLB_CIRCLE_NB 128                         // texel buckets per plane (n / 128 texels each)
#define GLB_TEXMM_STRIDE (2 + 2 * GLB_CIRCLE_NB)  // u32 per plane

// Full-plane K5 tap table (built once per parameter set, capi.cu): for every block of K5_BLOCK output texels the taps of
// all its texels, tap-major and padded to the block's longest sum with zero-weight entries, so a warp's loads coalesce
// and the tap loop is uniform.
struct K5Table {
    const int4*  blk;      // [n / K5_BLOCK] {first entry, taps per texel (padded), first input index, input span}
    const int2*  ent;      // entries {input index - first input index, weight bits}
    const float* wsum;     // [count] sum of an output's weights in loop order
    int smem_bytes;        // dynamic shared memory the kernel needs: planes per CTA * max span * sizeof(float)
    const int* out;        // [count] texel each output position writes (nullptr: position = texel, count = n)
    int count;             // outputs (need-list tables: the texels the module samples; full table: n)
    int max_span;
};
#ifndef K5_BLOCK
#define K5_BLOCK 128
#endif
// The spectrum path's device tables (capi.cu build_tables uploads the ones the plan names and owns them; null / 0 elsewhere)
struct SpectrumDevTables {
    int* need = nullptr; int need_count = 0;                  // lazy K5 need-list [2][need_count]
    TapEntry* tap_tab = nullptr; int* tap_cnt = nullptr; float* tap_wsum = nullptr; int tap_max = 0;   // its taps, tap-major
    // the same taps as one texel-major blob per channel (float w[] | u16 idx[] | int off[]), SpectrumArgs::csr
    unsigned char* csr = nullptr; int csr_bytes = 0, csr_idx_off = 0, csr_off_off = 0;
    void* need_blk = nullptr; int need_nblk = 0, need_max_rows = 0;   // k5_need_smem_kernel: blocks of sampled texels
    float* av_t = nullptr;                                    // k5_need_kernel: transposed pre-smoothing texels
    K5Table k5 = {};                                          // whole-plane K5 tap table (blk null: none)
};

// ---- kernel launchers (spectrum_kernels.cu, raster_kernels.cu); `stream` is a cudaStream_t passed as void* ------------------
struct SpectrumPlan;
// The spectrum-stream kernels of one modified update in the launch structure `plan` names (spectrum_plan.h): spectrum_kernel,
// then epilogue_b_kernel, then the need-list K5 kernel(s), then the whole-plane K5 unless a post chain follows (a.skip_tex:
// it runs after the upload).  `a` carries the per-update buffers and values, av_out = the pre-smoothing texture buffer; the
// launcher sets every field the plan decides.  Returns the number of kernels launched, or a negative error code.
int launch_spectrum_update(const glava_b200_params& p, const SpectrumPlan& plan, const SpectrumDevTables& tables,
                           const SpectrumArgs& a, void* stream);
// Whole-plane K5 over `count` R16 planes d_in -> d_out: k5_table_kernel from `table` with plan.table_planes planes per CTA
// when the plan has that table (plan.full_table; under K5Form::FULL_TABLE), else k5_planes_kernel (FULL_PLANES), whose
// refusal the caller checks (SpectrumPlan::refusal, k5_planes_refusal)
int launch_k5_full(const glava_b200_params& p, const SpectrumPlan& plan, const K5Table& table, const uint16_t* d_in,
                   uint16_t* d_out, int count, void* stream);
// the raster kernels of one pass (raster_plan.h plan_raster; texmm_kernel aside); p: the raster view (raster_view)
struct RasterPlan;
// A styled plan (plan.styled) reads the style slots from the RasterPass `a` is then part of.
int launch_raster(const glava_b200_params& p, const RasterPlan& plan, const RasterArgs& a, void* stream);
int launch_bars_rowtab(const glava_b200_params& p, void* d_rowtab, void* stream);
int launch_texmm(const glava_b200_params& p, const uint16_t* d_tex, uint32_t* d_out, int planes, void* stream);
// geometry cache of the polar modules over box = {x0, y0, w, h} (raster_plan.h polar_geo_box)
int launch_polar_geo(const glava_b200_params& p, void* d_geo, const int box[4], void* stream);
// circle: the per-tile texel reference ranges from the finished cache; d_tiles = int4[ntx * nty] followed by int[ntx * nty]
size_t circle_tile_bytes(const glava_b200_params& p, int* ntx, int* nty);
int launch_circle_tiles(const glava_b200_params& p, const void* d_geo, const int box[4], void* d_tiles, void* stream);
int launch_fifo_ingest(const glava_b200_params& p, const void* d_chunks, bool float_in, int frames, const float* src_l, const float* src_r,
                       float* dst_l, float* dst_r, int batch, void* stream);
int spectrum_threads(int n);
// chain_kernels.cu: optional stages of rd_update (bufscale, transform_smooth, keyframe lerp + R16 upload)
int launch_bufscale(const float* in_l, const float* in_r, float* out_l, float* out_r, int batch, int n_in, int k,
                    int channels, void* stream);
int launch_transform_smooth(float* d_planes, int n, const void* d_tab, int asz, int lim, int count, void* stream,
                            const uint32_t* d_umask = nullptr, int mask_shift = 1);   // d_umask: SpectrumArgs::umask, planes of unmodified
                            // streams are skipped; stream of plane i = i >> mask_shift (1: interleaved [batch*2] planes, 0: one channel's [batch])
int launch_upload(const float* d_s, const float* d_e, float mod, uint16_t* d_out, size_t total, void* stream);
// stream_state_kernels.cu: per-stream state <-> blob-ordered staging (stream_state_core.h); d_table = int stream[count]
// followed by uint32 cursor[count]; d_in == nullptr zeroes the streams' state
struct StateLayout; struct StatePtrs;
int launch_state_pack(const StateLayout& L, const StatePtrs& P, const int* d_table, int count, void* d_out, void* stream);
int launch_state_unpack(const StateLayout& L, const StatePtrs& P, const int* d_table, int count, const void* d_in, void* stream);
// export_kernels.cu: glava_b200_export_frames (DESIGN 4.10), one launch for the whole list.  The list ([count] entries)
// is in device memory; marks == nullptr (or mark_rows == 0) reads every framebuffer row, else only the rows the marks say
// may be non-zero (export_core.h)
struct alignas(16) ExportEntry {
    uint8_t* dst;               // the caller's destination
    int      slot;              // framebuffer slot of the listed stream (stream % slots)
    int      pad;
};
struct ExportArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // dirty-row marks of the last raster pass, or nullptr
    int             mark_rows;  // their band height
    const ExportEntry* list;
    int    count, w, h;
    int    format, over, native;  // export_core.h ExportFmt
    uint32_t bg;
    size_t pitch, uv_offset;    // uv_offset: luma to chroma plane (export_core.h ExportPlanes cb)
    size_t cr_offset;           // planar formats: Cb to Cr plane (ExportPlanes cr)
    int    enc;                 // Y'CbCr encoding, export_core.h export_enc of the flags (0: BT.709 limited range)
};
// NV12, RGBA and BGRA run export_kernel; I420, YUV444 and P010 export_yuv_kernel; any other encoding than 0 the kernels'
// instantiations for it (export_nv12_enc_kernel, export_yuv_enc_kernel); YUV420P10 and YUV444P10 export_p10_kernel;
// YUVA420P, YUVA444P10 and straight RGBA / BGRA (format: export_core.h export_kernel_format) export_yuva_kernel
int launch_export(const ExportArgs& a, void* stream);
// The entry of the scaled export and the overlay: ExportEntry with a chroma pointer, so that one call can fill an NV12
// mosaic, where each tile's chroma sits at a different offset from its luma
struct alignas(8) ExportEntryUV {
    uint8_t* dst;               // output row 0 (RGBA / BGRA pixels, or Y samples)
    uint8_t* dst_uv;            // NV12 / P010: CbCr row 0; planar formats: Cb row 0 (unused for RGBA / BGRA)
    int      slot;              // framebuffer slot of the listed stream
    int      pad;               // the overlay's fade kernel (DESIGN 4.20): the entry's opacity K, 1..255; else 0
};
// export_kernels.cu: glava_b200_export_scaled (DESIGN 4.11), one launch for the whole list, its own argument struct and
// ExportEntryUV entries so that export_kernel keeps its machine code.  Crop and output size are common to the list; d = src_w * src_h is
// divided by as export_core.h export_div with (div_mul, div_shift).
struct ScaledArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // as ExportArgs
    int             mark_rows;
    const ExportEntryUV* list;
    int    count, w, h;
    int    format, over, native;
    uint32_t bg;
    size_t pitch;
    int    src_x, src_y, src_w, src_h, out_w, out_h;   // crop in top-down coordinates, output size
    uint64_t div_mul;
    int    div_shift;
    size_t cr_offset;           // as ExportArgs
    int    enc;                 // as ExportArgs
};
// NV12, RGBA and BGRA run export_scaled_kernel; I420, YUV444 and P010 export_scaled_yuv_kernel; enc != 0 their
// instantiations for it (export_scaled_enc_kernel, export_scaled_yuv_enc_kernel); YUV420P10 and YUV444P10
// export_scaled_p10_kernel
int launch_export_scaled(const ScaledArgs& a, void* stream);
// export_kernels.cu: glava_b200_overlay_frames (DESIGN 4.12), one launch for the whole list, its own argument struct and
// ExportEntryUV entries.  band = 1 (native opacity with marks): one warp per (entry, band of mark_rows rows, strip), else one per
// (entry, output row pair, strip) as export_kernel.  An entry's dst is the rectangle's top-left pixel or Y byte.
struct OverlayArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // as ExportArgs
    int             mark_rows;
    const ExportEntryUV* list;
    int    count, w, h;
    int    format, native, band;
    size_t pitch;
    int    enc;                 // NV12: the destination's encoding, as ExportArgs (enc != 0 runs overlay_enc_kernel)
    int    fade;                // DESIGN 4.20: 1 runs overlay_fade_kernel, each entry's pad its opacity K (in what was padding)
};
int launch_overlay(const OverlayArgs& a, void* stream);
// export_kernels.cu: glava_b200_overlay_planes (DESIGN 4.17), one launch for the whole list.  Items as OverlayArgs'; an
// entry holds the rectangle's first sample in each plane (Y; CbCr for NV12 / P010, else Cb; Cr for the planar formats)
struct alignas(16) OverlayPlanesEntry {
    uint8_t* plane[3];
    int      slot;              // framebuffer slot of the listed stream
    int      pad;               // as ExportEntryUV's: the fade kernel's opacity K
};
struct OverlayPlanesArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // as ExportArgs
    int             mark_rows;
    const OverlayPlanesEntry* list;
    int    count, w, h;
    int    format, native, band;   // format: NV12, I420, YUV444, P010, YUV420P10 or YUV444P10
    size_t pitch, chroma_pitch;    // bytes between luma rows, between rows of every chroma plane
    int    enc;                 // the picture's encoding, as ExportArgs
    int    fade;                // as OverlayArgs: 1 runs overlay_planes_fade_kernel (in what was padding)
};
// overlay_planes_kernel (fade: overlay_planes_fade_kernel), instantiated per format, encoding, item kind and index width
int launch_overlay_planes(const OverlayPlanesArgs& a, void* stream);
// export_kernels.cu: glava_b200_overlay_scaled (DESIGN 4.21), one launch for the whole list: each entry's out_w x out_h
// rectangle gets export_scaled's pixel of the source rectangle (native: the premultiplied average; any other opacity: of
// opaque pixels), scaled by the entry's K (pad) and blended by the format's native body.  Entries as overlay_planes'
// (RGBA / BGRA: plane[0] only); w, h, marks and mark_rows describe the framebuffer as ScaledArgs' do.
struct OverlayScaledArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // as ExportArgs
    int             mark_rows;
    const OverlayPlanesEntry* list;
    int    count, w, h;
    int    format, native;      // format: RGBA, BGRA or one of overlay_planes'
    size_t pitch, chroma_pitch;    // as OverlayPlanesArgs (RGBA / BGRA: chroma_pitch 0)
    int    src_x, src_y, src_w, src_h, out_w, out_h;   // as ScaledArgs
    uint64_t div_mul;
    int    div_shift;
    int    enc;                 // as ExportArgs
};
// overlay_scaled_kernel, instantiated per format (RGBA and BGRA share one), encoding and index width
int launch_overlay_scaled(const OverlayScaledArgs& a, void* stream);
// export_kernels.cu: glava_b200_export_ladder (DESIGN 4.13), one launch for every rung of every entry.  Per rung what a
// standalone call would take: the whole frame at its own size (whole = 1) runs export_kernel's items, every other rung
// export_scaled_kernel's; z*: what a zero pixel becomes under the rung's format (export_core.h, filled on the host).
struct LadderRung {
    int    format, over, whole;
    uint32_t bg;
    size_t pitch;
    int    src_x, src_y, src_w, src_h, out_w, out_h;   // as ScaledArgs
    uint64_t div_mul;
    int    div_shift;
    uint32_t zpx, zy, zuv, zc;  // export_kernel's zpx / zy / zuv, export_scaled_kernel's zc
    int    enc;                 // as ExportArgs (in what was padding: the struct keeps its 80 bytes)
};
// The grid is flattened over (entry, unit of `sched`), the unit fastest; list: [count][nrungs] entries
struct LadderArgs {
    const uint8_t*  fb;         // [slots][h][w] RGBA8
    const uint32_t* marks;      // as ExportArgs
    int             mark_rows;
    const ExportEntryUV* list;
    int    count, w, h;
    int    native, nrungs;
    const uint64_t* sched;      // ladder_plan.h units, sorted by the first framebuffer row they read
    uint32_t units;
    LadderRung rung[GLAVA_B200_LADDER_MAX];
    // Y'CbCr rungs but NV12: the Cb to Cr distance (ExportArgs cr_offset) and export_core.h export_zero (planar 10-bit:
    // export_zero10) of the rung; alpha rungs export_zero_alpha, whose A word za sits in what was padding
    struct { size_t cr_offset; uint32_t zy, zu, zv, za; } yuv[GLAVA_B200_LADDER_MAX];
};
// export_ladder_kernel, or export_ladder_yuv_kernel when a rung is I420, YUV444 or P010, or export_ladder_enc_kernel when a
// rung has an encoding other than 0, or export_ladder_p10_kernel when a rung is YUV420P10 or YUV444P10
int launch_export_ladder(const LadderArgs& a, void* stream);
// capi.cu, for export.cpp: what the frame export reads of a renderer, and the slot where it keeps its own per-renderer
// state (*attach, released by *attach_free when the renderer is destroyed)
struct RendererView {
    bool built;
    int  device, batch, slots, w, h, native, mark_key;   // native: premultiply_alpha; mark_key: capi.cu's record of the marks
    void* stream;                                        // the raster stream (cudaStream_t)
    const uint8_t* fb; const uint32_t* marks;
    uint64_t* launches;
    void** attach; void (**attach_free)(void*);
};
RendererView renderer_view(glava_b200* r);
// export.cpp: the three caller-buffer exports, which differ in output size (the scaled export's is its rectangle's), the
// flags they take and their kernel
enum class ExportKind { frames, scaled, overlay, ladder };
// Every refusal of a call of `kind` that depends on this renderer alone, in the call's order (the overlay's overlap and
// framebuffer tests are overlay_geometry_check's); nothing is enqueued.  dst_uv and scale may be null; q (if non-null)
// receives the scale rectangle with its defaults applied, the whole frame for the other kinds.
int export_check(ExportKind kind, glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
                 const glava_b200_export* desc, const glava_b200_export_scale* scale, const char* who,
                 glava_b200_export_scale* q = nullptr);
// The call of `kind` on one renderer (glava_b200_export_frames / _export_scaled / glava_b200_overlay_frames): every check,
// then the list copy and the kernel on the raster stream behind `after_event` (or nothing), then `done_event` (or nothing).
// The overlay's `opacity` ([count] K, DESIGN 4.20; null: all 255) drops K = 0 entries and runs the fade kernel unless every K
// is 255; `who` (null: the plain call's name) names the call in its messages.
int export_run(ExportKind kind, glava_b200* r, const int* streams, int count, void* const* dst, void* const* dst_uv,
               const glava_b200_export* desc, const glava_b200_export_scale* scale, void* after_event, void* done_event,
               const uint8_t* opacity = nullptr, const char* who = nullptr);
// export_ladder.cpp, glava_b200_export_ladder: `rungs` non-null and 1 <= nrungs <= GLAVA_B200_LADDER_MAX (checked first, also by the sharded form
// before it splits the list); then export_check of the scaled kind once per rung, `who` extended by the rung's index; dst and
// dst_uv are [count][nrungs].  q (if non-null): [nrungs] rectangles with their defaults applied.
int ladder_shape_check(const glava_b200_export_rung* rungs, int nrungs, const char* who);
int ladder_check(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs, int nrungs, void* const* dst,
                 void* const* dst_uv, const char* who, glava_b200_export_scale* q = nullptr);
int ladder_run(glava_b200* r, const int* streams, int count, const glava_b200_export_rung* rungs, int nrungs, void* const* dst,
               void* const* dst_uv, void* after_event, void* done_event, const char* who);
// The rectangles of a list (w x h frames, `desc`'s format and pitch; dst_uv null: dst + uv_offset) must not overlap each
// other nor any of the `nfb` byte ranges [fb[k], fb[k] + fb_bytes[k]) (framebuffer arrays)
int overlay_geometry_check(int w, int h, int count, void* const* dst, void* const* dst_uv, const glava_b200_export& desc,
                           const uint8_t* const* fb, const size_t* fb_bytes, int nfb, const char* who);
// overlay_planes.cpp, glava_b200_overlay_planes (DESIGN 4.17).  planes_geometry: the descriptor against a w x h frame (format,
// flags, even 4:2:0 sizes, both pitches) and the planes' shapes; planes_check: every refusal that depends on this renderer
// alone (the overlap and framebuffer tests are planes_geometry_check's, over rectangles each with its own pitch P and row
// bytes B); planes_run: the call on one renderer.
// The scaled overlay (glava_b200_overlay_scaled, DESIGN 4.21) passes `q`, its rectangle with the defaults applied: the
// descriptor is then checked against q->out_w x q->out_h, and RGBA / BGRA are one plane of 4 bytes per pixel (chroma_pitch 0).
struct PlanesGeom { int planes; size_t luma_row, chroma_row; int chroma_rows; };
struct PlaneRect { uintptr_t p; size_t rows, P, B; int entry, plane; };
int planes_geometry(int w, int h, const glava_b200_overlay_planes_desc& d, PlanesGeom* g, const char* who, bool rgba = false);
int planes_check(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                 const glava_b200_overlay_planes_desc* desc, const char* who, const glava_b200_export_scale* q = nullptr);
bool plane_rects_meet(const PlaneRect& a, const PlaneRect& b);
int planes_geometry_check(int w, int h, int count, const glava_b200_picture* pics, const glava_b200_overlay_planes_desc& desc,
                          const uint8_t* const* fb, const size_t* fb_bytes, int nfb, const char* who, bool rgba = false);
int planes_run(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics, const glava_b200_overlay_planes_desc* desc,
               void* after_event, void* done_event, const char* who, const uint8_t* opacity = nullptr);
// export.cpp: the scale rectangle of export_scaled against a w x h frame (null, empty or leaving the frame, upscaling); *q
// receives it with the whole-frame default applied
int scale_check(int w, int h, const glava_b200_export_scale* s, glava_b200_export_scale* q, const char* who);
// overlay_scaled.cpp, glava_b200_overlay_scaled (DESIGN 4.21): the call on one renderer.  The whole frame at its own size runs
// export_run's / planes_run's overlay (its plain or fade kernel); any other rectangle overlay_scaled_kernel.
int scaled_overlay_run(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                       const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale, const uint8_t* opacity,
                       void* after_event, void* done_event, const char* who);
// the scaled overlay's checks that depend on one renderer alone (*q: the rectangle with its defaults applied)
int scaled_overlay_check(glava_b200* r, const int* streams, int count, const glava_b200_picture* pics,
                         const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                         glava_b200_export_scale* q, const char* who);
// capi.cu, for sharded.cpp: the blob checks of glava_b200_load_streams (nothing is touched), and save / load with one
// host pointer per listed stream (the blobs of one shard's streams are not contiguous in the caller's array)
int state_check_blobs(const glava_b200* r, const void* const* blobs, int count, const char* who);
int state_save_ptrs(glava_b200* r, const int* streams, int count, void* const* blobs);
int state_load_ptrs(glava_b200* r, const int* streams, int count, const void* const* blobs);

}  // namespace glb

#endif
