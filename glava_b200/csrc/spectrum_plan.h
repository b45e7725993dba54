// spectrum_plan.h — the launch structure of one spectrum update, chosen in one place (host only).
//
// One update of the spectrum path runs in one of several launch structures with identical arithmetic (DESIGN 4.1a): the
// pipeline-B epilogue inside spectrum_kernel or as epilogue_b_kernel; K5 inside spectrum_kernel (need-list taps from shared
// memory, from the L2 tap table or evaluated per tap; whole planes), as a need-list kernel (k5_need_smem_kernel, or
// av_transpose_kernel + k5_need_kernel) or as a whole-plane kernel (k5_table_kernel, k5_planes_kernel); the FFT pass
// variant; the persistent grid.  plan_spectrum makes every one of these choices from the effective parameters, the
// environment overrides (SpectrumKnobs) and the sizes of the host tables (tables.h).  capi.cu build_tables stores the plan
// on the handle and uploads the tables it names; spectrum_kernels.cu launch_spectrum_update executes it, run_update calls
// that once per modified update.  No CUDA here: tests/emul compiles the same decision for the host test tier.
#ifndef GLB_SPECTRUM_PLAN_H
#define GLB_SPECTRUM_PLAN_H

#include "tables.h"

#include <climits>
#include <cstdio>
#include <cstdlib>
#include <string>

namespace glb {

#ifndef K5_S_PLANES
#define K5_S_PLANES 8        // planes that share one tap (K5_S in spectrum_kernels.cu)
#endif
constexpr size_t K5_SMEM_MAX = 200 * 1024;             // dynamic shared memory the K5 kernels ask for at most

// spectrum_kernel's shared memory in place (SpecCfg): cpx buffer (also the raw-PCM staging area) | u16 av[n] | mbarriers
constexpr int spectrum_buf_bytes(int n) { return ((fft_padded_size(n / 2) * 8 + 15) / 16) * 16; }
constexpr int spectrum_smem_bytes(int n) { return spectrum_buf_bytes(n) + n * 2 + 16; }

// k5_planes_kernel: the widest input range a block of K5_BLOCK texels stages (scale_audio is increasing, so a block's taps
// lie between those of its first and last texel)
inline int k5_planes_span(const glava_b200_params& p) {
    const SmoothParams sp = smooth_params(p);
    const float fn = (float) p.n;
    int span = 0;
    for (int x0 = 0; x0 < p.n; x0 += K5_BLOCK) {
        const int x1 = (x0 + K5_BLOCK < p.n) ? x0 + K5_BLOCK : p.n;
        const float lo_f = scale_audio(sp, g_clamp(((float) x0 + 0.5f) / fn - sp.smooth_factor, 0.0f, 1.0f)) * fn;
        const float hi_f = scale_audio(sp, g_clamp(((float) (x1 - 1) + 0.5f) / fn + sp.smooth_factor, 0.0f, 1.0f)) * fn;
        int lo = (int) floorf(lo_f) - 2, hi = (int) ceilf(hi_f) + 3;
        lo = lo < 0 ? 0 : lo; hi = hi > p.n ? p.n : hi;
        if (hi - lo > span) span = hi - lo;
    }
    return span;
}
// its dynamic shared memory: K5_S_PLANES staged spans of u16 texels
inline size_t k5_planes_smem(int span) { return (size_t) K5_S_PLANES * (span > 0 ? span : 1) * sizeof(uint16_t); }
// the error k5_planes_kernel is refused with at that span ("" when its spans fit)
inline std::string k5_planes_refusal(int span) {
    if (k5_planes_smem(span) <= K5_SMEM_MAX) return std::string();
    char buf[96];
    snprintf(buf, sizeof(buf), "smooth pass: tap span %d too large for shared memory", span);
    return buf;
}
// k5_table_kernel: planes per CTA that share every tap load, as many as the staged float spans leave room for
inline int k5_table_planes(int max_span) {
    const size_t per_plane = (size_t) max_span * sizeof(float);
    return 8 * per_plane <= K5_SMEM_MAX ? 8 : (4 * per_plane <= K5_SMEM_MAX ? 4 : 2);
}

// ---- environment overrides (GLAVA_B200_<name>, DESIGN 6.2) ------------------------------------------------------------
constexpr int KNOB_UNSET = INT_MIN;
struct SpectrumKnobs {
    int  tap_ku = 8;                    // TAP_KU: L2 tap-table entries a thread keeps in flight
    bool fused_k5 = false;              // FUSED_K5: whole-plane K5 inside spectrum_kernel
    bool split_epi = true;              // SPLIT_EPI=0: the pipeline-B epilogue stays inside spectrum_kernel
    int  spec_oop = KNOB_UNSET;         // SPEC_OOP: out-of-place FFT passes (unset: the size's default)
    int  spec_t = KNOB_UNSET;           // SPEC_T: spectrum CTA size (unset: the size's default)
    int  spec_ctas_per_sm = KNOB_UNSET; // SPEC_CTAS_PER_SM: persistent spectrum CTAs per SM (0: one CTA per work unit)
    int  spec_resident = 0;             // SPEC_RESIDENT: resident spectrum CTAs per SM, capped through shared memory (0: no cap)
    bool no_epi_prune = false;          // NO_EPI_PRUNE: the lazy epilogue runs over every bin
    bool no_taptab = false;             // NO_TAPTAB: need-list K5 evaluates its taps in the kernel
    bool no_smem_taps = false;          // NO_SMEM_TAPS: the in-kernel need-list K5 reads its taps through L2
    int  k5_split = -1;                 // K5_SPLIT=0|1: need-list K5 as its own kernel off / on (-1: by size)
    bool k5n_smem = true;               // K5N_SMEM=0: that kernel reads through L2 (k5_need_kernel) instead of tiles
    int  k5n_rows = -105;               // K5N_ROWS: tile rows, or -per cent of the tallest window (tables.h build_need_blocks)
    int  k5n_tpb = 16;                  // K5N_TPB: sampled texels per tile
    int  k5n_s = 0;                     // K5N_S=1|2|4: streams per lane of k5_need_kernel (0: by batch)
    int  k5n_warps = 0;                 // K5N_WARPS=1..16: warps per CTA of the need-list kernels (0: their default)
    bool no_k5_table = false;           // NO_K5_TABLE: whole-plane K5 evaluates its taps in the kernel
};

// `get(name)`: the value of the variable GLAVA_B200_<...> or nullptr (getenv in the library, a dictionary in the host build).
// A value outside a knob's range leaves its default.
template <class Get>
SpectrumKnobs spectrum_knobs(Get get) {
    SpectrumKnobs k;
    const char* e;
    auto num = [&](const char* name, int* out) { if ((e = get(name))) *out = atoi(e); };
    num("GLAVA_B200_TAP_KU", &k.tap_ku);
    k.fused_k5 = get("GLAVA_B200_FUSED_K5") != nullptr;
    if ((e = get("GLAVA_B200_SPLIT_EPI"))) k.split_epi = atoi(e) != 0;
    num("GLAVA_B200_SPEC_OOP", &k.spec_oop);
    num("GLAVA_B200_SPEC_T", &k.spec_t);
    num("GLAVA_B200_SPEC_CTAS_PER_SM", &k.spec_ctas_per_sm);
    num("GLAVA_B200_SPEC_RESIDENT", &k.spec_resident);
    k.no_epi_prune = get("GLAVA_B200_NO_EPI_PRUNE") != nullptr;
    k.no_taptab = get("GLAVA_B200_NO_TAPTAB") != nullptr;
    k.no_smem_taps = get("GLAVA_B200_NO_SMEM_TAPS") != nullptr;
    if ((e = get("GLAVA_B200_K5_SPLIT"))) k.k5_split = atoi(e) != 0;
    if ((e = get("GLAVA_B200_K5N_SMEM"))) k.k5n_smem = atoi(e) != 0;
    if ((e = get("GLAVA_B200_K5N_ROWS"))) { const int v = atoi(e); if (v >= 32 || v < 0) k.k5n_rows = v; }
    if ((e = get("GLAVA_B200_K5N_TPB"))) { const int v = atoi(e); if (v >= 1) k.k5n_tpb = v; }
    if ((e = get("GLAVA_B200_K5N_S"))) { const int v = atoi(e); if (v == 1 || v == 2 || v == 4) k.k5n_s = v; }
    if ((e = get("GLAVA_B200_K5N_WARPS"))) { const int v = atoi(e); if (v >= 1 && v <= 16) k.k5n_warps = v; }
    k.no_k5_table = get("GLAVA_B200_NO_K5_TABLE") != nullptr;
    return k;
}

// ---- the plan -----------------------------------------------------------------------------------------------------------
enum class K5Form {
    NONE,            // smooth pass off
    TAPS_SMEM,       // need-list K5 inside spectrum_kernel, taps from the texel-major blob in shared memory
    TAPS_L2,         // the same from the tap-major table through L2, tap_ku entries in flight
    TAPS_DIRECT,     // the same with every tap evaluated in the kernel (no tap table)
    NEED_SMEM,       // need-list K5 as k5_need_smem_kernel (tiles of sampled texels)
    NEED_L2,         // need-list K5 as av_transpose_kernel + k5_need_kernel (k5n_s streams per lane)
    FULL_TABLE,      // whole planes as k5_table_kernel (table_planes planes per CTA)
    FULL_PLANES,     // whole planes as k5_planes_kernel (taps evaluated in the kernel)
    FUSED,           // whole planes inside spectrum_kernel
};

struct SpectrumPlan {
    // the tables build_tables uploads
    bool need_list = false;        // need-list (lazy K5)
    bool tap_table = false;        // its tap-major table and texel-major blob
    bool full_table = false;       // the whole-plane K5 table (glava_b200_smooth_pass reads it too)
    // the launches
    bool split_epilogue = false;   // pipeline B: spectrum_kernel stops after the FFT (fft_only), epilogue_b_kernel follows
    int  epi_n = 0;                // SpectrumArgs::epi_n: bins the epilogue runs over (0: all; split: a multiple of 8)
    int  av_t_len = 0;             // need-list kernels: leading bins of the pre-smoothing texture they read
    K5Form k5 = K5Form::NONE;      // where K5 runs; with a post chain the whole-plane forms follow the upload
    int  tap_ku = 8;               // SpectrumArgs::tap_ku
    int  table_planes = 0;         // full_table: planes per k5_table_kernel CTA (FULL_TABLE, glava_b200_smooth_pass)
    int  k5n_s = 0;                // NEED_L2: streams per lane
    int  k5n_warps = 0;            // NEED_SMEM, NEED_L2: warps per CTA
    int  fft_oop = 0, fft_t = 0;   // FFT pass variant: out of place, threads per CTA (0: the size's default)
    int  spec_grid = 0;            // spectrum_kernel CTAs (fewer than work units: persistent)
    int  spec_resident = 0;        // resident spectrum CTAs per SM it is capped at (0: no cap)
    std::string refusal;           // non-empty: every update with a new texture fails with this error before it enqueues anything
};

// The host tables a plan is computed from, each built the first time the decision reads it (the whole-plane table takes
// seconds for wide windows at 16384); build_tables uploads the ones the plan names.
struct SpectrumTables {
    bool need = false;             // a need-list exists: `lazy` holds it and its taps
    LazyTables lazy;
    NeedBlocks blocks;             // tiles of sampled texels (need-list K5 as its own kernel)
    K5TableHost full;              // taps of every texel (whole-plane K5 outside spectrum_kernel)
};

// p: the effective parameters (n = setbufsize / setbufscale); post_chain: transform_smooth / keyframe interpolation follow
// the spectrum kernel as their own kernels; sm_count: of the device the handle runs on.
inline SpectrumPlan plan_spectrum(const glava_b200_params& p, bool post_chain, int batch, int sm_count, const SpectrumKnobs& k,
                                  SpectrumTables* t) {
    SpectrumPlan pl;
    const int n = p.n;
    const bool is_fft = p.module != GLAVA_B200_MOD_WAVE;
    pl.tap_ku = k.tap_ku;
    // FFT pass variant: out of place with 256 threads at 8192, the measured optimum (tools/variant_sweep.sh)
    pl.fft_oop = k.spec_oop != KNOB_UNSET ? k.spec_oop : (n == 8192 ? 1 : 0);
    pl.fft_t = k.spec_t != KNOB_UNSET ? k.spec_t : (n == 8192 ? 256 : 0);
    if (p.smooth_pass && p.lazy_smooth && !post_chain) {
        std::vector<int> lists[2];
        if (build_need_list(p, lists)) { t->need = true; build_lazy_tables(p, lists, &t->lazy); }
    }
    if (t->need) {
        const LazyTables& lt = t->lazy;
        pl.need_list = true;
        pl.epi_n = k.no_epi_prune ? 0 : lt.epi_n;
        pl.tap_table = lt.tab.size() * sizeof(TapEntry) <= (size_t) 64 << 20 && !k.no_taptab;
        pl.k5 = K5Form::TAPS_DIRECT;
        bool split = false;
        if (pl.tap_table) {
            // When one channel's blob is small enough for two CTAs per SM to hold it in shared memory next to the FFT
            // buffers, the kernel's serial per-texel sums read their taps from there (no L2 round trips on the chain).
            const bool fits = spectrum_smem_bytes(n) + lt.blob <= (size_t) 112 * 1024 && !k.no_smem_taps;
            pl.k5 = fits ? K5Form::TAPS_SMEM : K5Form::TAPS_L2;
            // Need-list K5 as its own kernel (lanes = streams): whenever the taps do not fit shared memory next to the FFT,
            // and from setbufsize 4096 up anyway
            split = k.k5_split >= 0 ? k.k5_split != 0 : (!fits || n >= 4096);
        }
        if (split) {
            pl.av_t_len = lt.epi_n > 0 ? lt.epi_n : n;
            build_need_blocks(lt, n, k.k5n_rows, k.k5n_tpb, &t->blocks);
            if (t->blocks.nblk > 0 && (size_t) t->blocks.max_rows * 33 * sizeof(float) <= K5_SMEM_MAX && k.k5n_smem) {
                pl.k5 = K5Form::NEED_SMEM;
                pl.k5n_warps = k.k5n_warps ? k.k5n_warps : 16;
            } else {
                pl.k5 = K5Form::NEED_L2;
                // 2 streams per lane share every tap broadcast once the batch is large enough to still fill the device;
                // with few sampled texels (radial: ~90 per channel) they do not fill it: one stream per lane there
                const long long channels = is_fft ? 2 : 1;
                pl.k5n_s = k.k5n_s ? k.k5n_s
                                   : (batch >= 256 && channels * (long long) lt.cnt * ((batch + 63) / 64) >= (long long) sm_count * 24 ? 2 : 1);
                pl.k5n_warps = k.k5n_warps ? k.k5n_warps : 4;
            }
            // and the R16 state update as its own elementwise kernel over the leading epi_n bins, rounded up to 8
            const int epi8 = ((pl.epi_n + 7) / 8) * 8;
            if (is_fft && p.accel_fft && k.split_epi && epi8 > 0 && epi8 <= n) { pl.split_epilogue = true; pl.epi_n = epi8; }
        }
    } else if (p.smooth_pass) {
        if (!k.no_k5_table) {
            build_k5_table_host(p, &t->full);
            pl.full_table = 2 * t->full.max_span * sizeof(float) <= K5_SMEM_MAX && t->full.ent.size() * sizeof(K5Ent) <= (size_t) 256 << 20;
            if (pl.full_table) pl.table_planes = k5_table_planes(t->full.max_span);
        }
        if (k.fused_k5 && !post_chain) pl.k5 = K5Form::FUSED;
        else if (pl.full_table) pl.k5 = K5Form::FULL_TABLE;
        else { pl.k5 = K5Form::FULL_PLANES; pl.refusal = k5_planes_refusal(k5_planes_span(p)); }
    }
    // Persistent grid: a few CTAs per SM.  Small on purpose: the kernel is latency bound and is meant to run UNDER the
    // HBM-bound raster kernel of the previous update without taking its occupancy away.  Global-memory taps: one CTA per
    // unit.  Shared-memory taps: 2 CTAs per SM (the kernel's residency) load the table once per CTA and let the TMA engine
    // prefetch the next unit's PCM during K5; an even grid keeps a CTA on one channel (one tap-table load).
    const bool csr = pl.k5 == K5Form::TAPS_SMEM;
    const int per_sm = k.spec_ctas_per_sm != KNOB_UNSET ? k.spec_ctas_per_sm : (csr ? 2 : 0);
    const int units = is_fft ? batch * 2 : batch;
    pl.spec_grid = (per_sm > 0 && sm_count * per_sm < units) ? sm_count * per_sm : units;
    if (csr && is_fft && pl.spec_grid < units && (pl.spec_grid & 1)) ++pl.spec_grid;
    pl.spec_resident = k.spec_resident;
    return pl;
}

}  // namespace glb

#endif
