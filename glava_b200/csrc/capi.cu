// capi.cu — the C ABI of include/glava_b200.h: renderer handle, device memory, streams.
//
// Plays the role of rd_new / rd_update / rd_destroy (reference glava/render.c:867,1743,2456)
// for a batch of independent streams on one CUDA device.  All device state (PCM staging,
// gravity/average state per stream and channel, R16 textures, framebuffers) is allocated once
// in glava_b200_new and stays resident in HBM.
#include "internal.h"
#include "raster_core.h"
#include "chain_core.h"
#include "tables.h"
#include "spectrum_plan.h"
#include "raster_plan.h"
#include "stream_state_core.h"
#include "cuda_owner.h"

#include <cuda_runtime.h>

#include <atomic>
#include <map>
#include <mutex>
#include <sched.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace glb {

// ---- error plumbing -----------------------------------------------------------------------------
static thread_local std::string g_last_error;
static thread_local bool g_has_error = false;
static void default_hook(const char* msg) { fprintf(stderr, "glava_b200: %s\n", msg); }
static void (*g_hook)(const char*) = default_hook;

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_last_error = buf; g_has_error = true;
    if (g_hook) g_hook(buf);
    return code;
}
void clear_error() { g_has_error = false; }
bool has_error() { return g_has_error; }

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

}  // namespace glb

using namespace glb;

// Everything build_tables derives from the parameters alone (audio-independent), released and rebuilt together on every
// reconfigure and resize: the launch structure of the spectrum update and the tables it reads, the row table, the polar
// geometry cache and circle tiles, the transform_smooth window table.  The raw pointers are views of `bufs`; null / 0
// where the configuration has none.
struct ConfigTables {
    SpectrumPlan plan;                                        // launch structure of the spectrum update (spectrum_plan.h)
    SpectrumDevTables spec;                                   // the K5 tables the spectrum plan names (internal.h)
    RasterTables raster;                                      // which raster tables exist (raster_plan.h), the cache's box
    void* rowtab = nullptr;                                   // bars / graph row colours, [h] {fill, outline} RGBA8 pairs
    void* geo = nullptr;                                      // polar geometry cache (radial / circle), see raster_kernels.cu
    void* ctile = nullptr; int ctile_nx = 0, ctile_count = 0; // circle: per-tile texel reference ranges (launch_circle_tiles)
    void* ts_tab = nullptr; int ts_asz = 0, ts_lim = 0;       // transform_smooth {smin, smax} table
    // stream styles (DESIGN 4.9), when any stream has one: the style slot of every stream [batch] and the slots' records
    // (RasterArgs::style_of / styles); rowtab then holds a table per slot, geo a radial cache per distinct (fg, bg)
    const int* style_of = nullptr; const StyleSlot* styles = nullptr;
    std::vector<DevBuf<>> bufs;
};

// The buffers sized by the frame, replaced on a resize: column table (graph / wave; the module of a handle never changes:
// reconfigure refuses), framebuffers [slots][h][w] RGBA8 and their dirty-row marks
struct FrameBuffers {
    DevBuf<float> coltab;       // graph / wave: per-stream column table (launch_raster fills it)
    DevBuf<uint8_t> fb;
    DevBuf<uint32_t> marks;     // dirty-row marks of the framebuffer slots (RasterArgs::marks)
};

// A parameter set as given, its effective parameters and mode flags, and the transform_average weights of every update
struct Derived {
    glava_b200_params user;     // as given (glava_b200_get_params)
    glava_b200_params p;        // n = setbufsize / setbufscale, accel_fft cleared when a transform follows "fft" (render.c:2143-2154)
    int n_in;                   // setbufsize: floats per channel the caller hands to glava_b200_update
    bool interp_on;             // keyframe interpolation active (render.c:1761-1763, 2161-2168)
    bool post_chain;            // transform_smooth and / or keyframe lerp: the spectrum kernel stops at the float chain
                                // result; upload + K5 run as separate kernels
    SpectrumArgs spec_args;     // what every update's SpectrumArgs starts from: the transform_average weights, all else 0
};

static Derived derive(const glava_b200_params& user) {
    Derived d{};
    d.user = user;
    d.p = user;
    d.n_in = user.n;
    d.p.n = user.n / user.bufscale;
    const bool is_fft = d.p.module != GLAVA_B200_MOD_WAVE;
    if (d.p.transform_smooth == 1 && is_fft) d.p.accel_fft = 0;           // (2 = "smooth" before "fft": applied to the PCM)
    const float fr = d.p.fr > 0.0f ? d.p.fr : d.p.ur;
    d.interp_on = d.p.interpolate && !(d.p.accel_fft && is_fft) && (d.p.ur / fr) <= 0.9f;
    d.post_chain = d.p.transform_smooth == 1 || d.interp_on;
    const int F = d.p.avg_frames;
    for (int f = 0; f < F; ++f) {
        // pipeline A: window_frame(f, avg_frames - 1) -> cos(TWOPI*f/F - 1), double (render.c:661,766)
        d.spec_args.avg_w_a[f] = 0.6 - (0.4 * cos(6.28318530718 * (double) f / (double) F - 1));
        // pipeline B: window(I, _AVG_FRAMES - 1) -> cos(TWOPI*I/F - 1), GLSL float (average_pass.frag:41)
        d.spec_args.avg_w_b[f] = 0.53836f - (0.46164f * cosf(6.28318530718f * (float) f / (float) F - 1.0f));
    }
    d.spec_args.avg_b_windowed = (d.p.avg_window && F != 2) ? 1 : 0;
    return d;
}

// Every member that holds a CUDA resource owns it; glava_b200_destroy synchronises the streams before the destructors run.
struct glava_b200 {
    Derived d;                  // the parameters of the last successful build (rebuild); the kernels run with d.p
    int  kcounter = 0;          // frames since the last modified update (render.c:2380-2383)
    DevBuf<float> d_scaled[2];  // bufscale output [batch][n] x {l, r}
    DevBuf<float> d_key[3]; int key_start = 0, key_end = 1;   // keyframe buffers [batch*2][n] (start, end, the one being written)
    float* d_spec_cur = nullptr;   // latest post-transform buffer (glava_b200_spectrum)
    std::atomic<unsigned long long> sizereq{0};   // pending glava_b200_sizereq: (1 << 63) | w << 32 | h, 0 = none
    int batch = 0, device = 0, slots = 0;
    Stream stream;                        // raster kernels, read-backs (the stream glava_b200_cuda_stream returns)
    Stream own_spec_stream;               // spec_stream unless GLAVA_B200_NO_OVERLAP makes it `stream`
    cudaStream_t spec_stream = nullptr;   // spectrum kernels + FIFO ingest, lowest priority: the latency-bound spectrum
                                          // kernel of update i+1 runs under the HBM-bound raster kernel of update i
    int    tex_cur = 0;         // which half of d_tex the latest spectrum wrote / the raster reads
    Event ev_spec_done[2], ev_raster_done[2];
    // inputs
    DevBuf<float> d_pcm[2][2];  // H2D staging for glava_b200_update, double-buffered  [2][batch][n] x {l, r}
    int    stage_cur = 0;
    Event ev_input;             // glava_b200_input_event
    bool   async_input = false; int last_in = -1;   // glava_b200_set_async_input: update() does not wait for its H2D copy
    Stream copy_stream;         // H2D of update i+1 overlaps the kernels of update i
    // asynchronous frame read-back: D2D into a staging frame on the raster stream (microseconds), D2H from there on its
    // own stream — the PCIe copy of frame i runs under raster i+1 instead of in front of it
    Stream out_stream; DevBuf<uint8_t> d_stage[2]; size_t stage_bytes = 0; int out_cur = 0;
    Event ev_stage_ready[2], ev_stage_free[2];
    Event ev_copied[2], ev_free[2];
    DevBuf<float> d_ring[2][2]; // FIFO rings, ping-pong                      [2][batch][n] x {l, r}
    int    ring_cur = 0;
    DevBuf<> d_chunks; size_t chunks_cap = 0;
    // constants
    DevBuf<double> d_window; DevBuf<float> d_twiddle;
    bool built = false;         // tab and frame hold a complete build for p (false after a failed reconfigure or resize)
    ConfigTables tab;           // build_tables
    FrameBuffers frame;
    DevBuf<uint32_t> d_texmm;   // circle: per-plane {min, max} of the sampled texture, refreshed before each raster
    // state + outputs
    DevBuf<float> d_spec;
    DevBuf<char> d_state;       // gravity + average state: the two views below, one allocation
    float* d_applied = nullptr; float* d_ring_f = nullptr; uint16_t* d_gr_store = nullptr; uint16_t* d_ring_u = nullptr;
    DevBuf<uint16_t> d_tex;
    DevBuf<uint16_t> d_av;      // pre-smoothing textures [batch*2][n] (full-plane K5 runs as its own kernel)
    // the launch structure that last wrote the dirty-row marks (RasterPlan::mark_key; 0 = none: the next bars / graph / wave
    // launch stores every row)
    int mark_key = 0;
    // per-stream styles as set (glava_b200_set_stream_styles), [batch]; empty: no stream has one
    std::vector<glava_b200_stream_style> styles;
    unsigned long long updates = 0;
    // per-stream `modified` masks (glava_b200_update_masked): once streams have advanced unevenly, every stream has its
    // own average-ring cursor; words {bit 31 = modified, low bits = cursor} go to the device through a small pinned ring
    bool desync = false;
    std::vector<uint32_t> cursor;          // [batch] modified updates of that stream so far, mod avg_frames (valid once desync)
    PinnedBuf<uint32_t> h_umask[4]; DevBuf<uint32_t> d_umask[4]; Event ev_umask[4]; int umask_cur = 0;
    // per-stream state I/O (glava_b200_save_streams / _load_streams / _reset_streams): two device staging halves, each
    // [chunk table: int stream[k], uint32 cursor[k]][blob segments of k streams], allocated on first use; the tables go up
    // from pinned host buffers.  ev_sst_copied[i]: the H2D copies into half i are done; ev_sst_free[i]: its kernel and D2H
    // copies are done
    DevBuf<char> d_sst[2]; PinnedBuf<int> h_sst[2]; Event ev_sst_copied[2], ev_sst_free[2];
    int sst_cur = 0, sst_streams = 0; size_t sst_table = 0;
    // state another source file keeps per renderer (export.cpp: the frame export's list buffers), created on its first use
    // through renderer_view and released by attach_free once the streams are drained (glava_b200_destroy)
    void* attach = nullptr; void (*attach_free)(void*) = nullptr;
    uint64_t launches = 0;
    // optional per-kernel device timing (glava_b200_set_timing): events around each launch
    bool timing = false;
    std::vector<Event> ev_spec; // pairs around each spectrum launch (spec_stream)
    std::vector<Event> ev_ras;  // pairs around each raster launch (stream)
};

// dirty-row marks: one word per (slot, row, 128-pixel strip), so that any band height finds its band's word at its first row
static size_t mark_bytes(const glava_b200_params& p, int slots) {
    return (size_t) slots * p.h * ((p.w + 127) / 128) * sizeof(uint32_t);
}

// A device buffer of `bytes`, zero-filled on `st`
template <typename T>
static int alloc_zeroed(DevBuf<T>& b, size_t bytes, cudaStream_t st) {
    int rc = b.alloc(bytes);
    if (rc) return rc;
    CU(cudaMemsetAsync(b, 0, bytes ? bytes : 16, st));
    return 0;
}

// A new device buffer of `bytes` owned by `tb`, *view pointing at it: filled from host memory `src` on `st`, zero-filled
// (`zero`), or left for a kernel to fill
template <typename T>
static int table_buf(ConfigTables& tb, T** view, size_t bytes, cudaStream_t st, const void* src, bool zero = false) {
    DevBuf<> b;
    int rc = zero ? alloc_zeroed(b, bytes, st) : b.alloc(bytes);
    if (rc) return rc;
    if (src && bytes) CU(cudaMemcpyAsync(b, src, bytes, cudaMemcpyHostToDevice, st));
    *view = (T*) b.get();
    tb.bufs.push_back(std::move(b));
    return 0;
}

extern "C" {

void glava_b200_set_abort_hook(void (*hook)(const char*)) { g_hook = hook ? hook : default_hook; }
const char* glava_b200_last_error(void) { return g_last_error.c_str(); }
const char* glava_b200_version(void) { return "glava_b200 0.1 (sm_90a)"; }

int glava_b200_default_params(glava_b200_params* out, const char* module) {
    clear_error();
    if (!out || !module) return fail(GLAVA_B200_EINVAL, "null argument");
    int m = module_from_name(module);
    if (m < 0) return fail(GLAVA_B200_ECONFIG, "Could not find module '%s'", module);
    fill_defaults(out, m);
    return GLAVA_B200_OK;
}

int glava_b200_load_config(glava_b200_params* out, const char* const* paths, const char* entry,
                           const char* const* requests, const char* force_module) {
    if (!out) return fail(GLAVA_B200_EINVAL, "null argument");
    return load_config(out, paths, entry, requests, force_module, nullptr);
}

int glava_b200_load_config_binds(glava_b200_params* out, const char* const* paths, const char* entry,
                                 const char* const* requests, const char* force_module, const char* const* binds) {
    if (!out) return fail(GLAVA_B200_EINVAL, "null argument");
    return load_config(out, paths, entry, requests, force_module, binds);
}

// ---- NUMA placement of pinned host memory -----------------------------------------------------------------------------
// On a two-socket box (e.g. an 8-GPU node with GPUs 0-3 behind socket 0, 4-7 behind socket 1) a pinned buffer on the other
// socket makes every H2D / D2H DMA cross the inter-socket link; eight ranks doing so together was what collapsed round 1's
// end-to-end scaling.  Pinned buffers are therefore page-placed on the NUMA node of the device they feed: anonymous
// mapping + mbind(MPOL_BIND) + first touch + cudaHostRegister.  No libnuma in the image: the raw syscall.
static std::mutex g_host_mu;
static std::map<void*, size_t> g_host_maps;          // mmap'd + registered blocks (everything else came from cudaHostAlloc)

static int device_numa_node(int device) {
    char bus[32] = { 0 };
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* c = bus; *c; ++c) if (*c >= 'A' && *c <= 'Z') *c = (char) (*c - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

extern "C" {

int glava_b200_device_numa_node(int device) { return device_numa_node(device); }
int glava_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// Pin the calling thread to the CPUs of the device's NUMA node (what `numactl --cpunodebind` does for a one-rank-per-GPU
// process).  Returns the node, or -1 when the topology is not exposed (nothing changed).
int glava_b200_bind_thread_to_device(int device) {
    const int node = device_numa_node(device);
    if (node < 0) return -1;
    char path[128];
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    cpu_set_t set; CPU_ZERO(&set);
    int a = 0, b = 0, any = 0;
    while (fscanf(f, "%d", &a) == 1) {
        b = a;
        int ch = fgetc(f);
        if (ch == '-') { if (fscanf(f, "%d", &b) != 1) b = a; ch = fgetc(f); }
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET(c, &set); any = 1; }
        if (ch != ',') break;
    }
    fclose(f);
    if (!any || sched_setaffinity(0, sizeof(set), &set) != 0) return -1;
    return node;
}

void* glava_b200_host_alloc_on(size_t bytes, int device) {
    if (bytes == 0) bytes = 16;
    const int node = getenv("GLAVA_B200_NO_NUMA") ? -1 : device_numa_node(device);
    if (node >= 0 && node < 64) {
        const size_t page = (size_t) sysconf(_SC_PAGESIZE);
        const size_t len = (bytes + page - 1) / page * page;
        void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (p != MAP_FAILED) {
            unsigned long mask = 1ul << node;
            const long rc = syscall(SYS_mbind, p, len, 2 /* MPOL_BIND */, &mask, 64ul, 0u);
            if (rc == 0) {
                for (size_t o = 0; o < len; o += page) ((volatile char*) p)[o] = 0;      // first touch: the pages now exist on `node`
                if (cudaHostRegister(p, len, cudaHostRegisterPortable) == cudaSuccess) {
                    std::lock_guard<std::mutex> lk(g_host_mu);
                    g_host_maps[p] = len;
                    return p;
                }
                cudaGetLastError();
            }
            munmap(p, len);
        }
    }
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        fail(GLAVA_B200_ECUDA, "cudaHostAlloc(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
void* glava_b200_host_alloc(size_t bytes) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    return glava_b200_host_alloc_on(bytes, dev);
}
void glava_b200_host_free(void* p) {
    if (!p) return;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> lk(g_host_mu);
        auto it = g_host_maps.find(p);
        if (it != g_host_maps.end()) { len = it->second; g_host_maps.erase(it); }
    }
    if (len) { cudaHostUnregister(p); munmap(p, len); }
    else cudaFreeHost(p);
}

}  // extern "C"

// ---- stream styles (DESIGN 4.9) ------------------------------------------------------------------------------------------
// The fields a style replaces (glava_b200_stream_style), and the refusals that do not need validate_params
static int style_fields(const glava_b200_params& base, const glava_b200_stream_style& s, glava_b200_params* q) {
    auto bad = [](const char* why) { return fail(GLAVA_B200_EINVAL, "stream style: %s", why); };
    if (s.set & ~(GLAVA_B200_STYLE_AMPLIFY | GLAVA_B200_STYLE_FG | GLAVA_B200_STYLE_BG)) return bad("unknown bits in `set`");
    *q = base;
    if (!s.set) return 0;
    const int m = base.module;
    if (m == GLAVA_B200_MOD_TEST) return bad("the test module has no AMPLIFY, @fg or @bg");
    if (s.set & GLAVA_B200_STYLE_AMPLIFY) {
        if (!std::isfinite(s.amplify)) return bad("amplify must be finite");
        *style_amplify_field(*q) = s.amplify;
    }
    if (s.set & GLAVA_B200_STYLE_FG) {
        if (s.fg.mode != 0 && s.fg.mode != 1) return bad("fg must be a constant (mode 1) or a gradient (mode 0)");
        if ((m == GLAVA_B200_MOD_CIRCLE || m == GLAVA_B200_MOD_WAVE) && s.fg.mode != 1)
            return bad("circle / wave take a constant fg (mode 1)");
        if (m == GLAVA_B200_MOD_BARS && !(s.set & GLAVA_B200_STYLE_BG) && base.bars_outline_mode == 2)
            return bad("fg without bg on bars whose BAR_OUTLINE is an expression (it was compiled against the renderer's COLOR)");
        // a constant, as the config reader stores a constant COLOR: hi = lo, the gradient stays
        auto take = [&](glava_b200_color* c, glava_b200_color_prog* prog) {
            const float g = c->gradient;
            *c = s.fg;
            if (c->mode == 1) { memcpy(c->hi, c->lo, sizeof(c->hi)); c->gradient = g; }
            prog->n_ops = 0;
        };
        switch (m) {
            case GLAVA_B200_MOD_BARS: take(&q->bars_color, &q->bars_color_prog); break;
            case GLAVA_B200_MOD_RADIAL: take(&q->radial_color, &q->radial_color_prog); break;
            case GLAVA_B200_MOD_GRAPH: take(&q->graph_color, &q->graph_color_prog); break;
            case GLAVA_B200_MOD_CIRCLE: memcpy(q->circle_outline, s.fg.lo, sizeof(q->circle_outline)); break;
            case GLAVA_B200_MOD_WAVE: memcpy(q->wave_base_color, s.fg.lo, sizeof(q->wave_base_color)); break;
        }
    }
    if (s.set & GLAVA_B200_STYLE_BG) {
        const size_t c4 = 4 * sizeof(float);
        switch (m) {
            case GLAVA_B200_MOD_BARS: q->bars_outline_mode = 1; memcpy(q->bars_outline, s.bg, c4); break;
            case GLAVA_B200_MOD_RADIAL: memcpy(q->radial_outline, s.bg, c4); memcpy(q->radial_bar_outline, s.bg, c4); break;
            case GLAVA_B200_MOD_GRAPH: memcpy(q->graph_outline, s.bg, c4); break;
            case GLAVA_B200_MOD_WAVE: memcpy(q->wave_outline, s.bg, c4); break;
            case GLAVA_B200_MOD_CIRCLE: return bad("circle has no @bg");
        }
    }
    return 0;
}

}  // extern "C"

namespace glb {
int style_apply(const glava_b200_params& base, const glava_b200_stream_style& s, glava_b200_params* out) {
    glava_b200_params q;
    int rc = style_fields(base, s, &q);
    if (rc) return rc;
    if ((rc = validate_params(&q)) != 0) return rc;
    *out = q;
    return 0;
}
}  // namespace glb

extern "C" {

// A style with only what it sets, so that equal looks compare equal byte for byte (a constant fg: lo alone)
static glava_b200_stream_style style_key(const glava_b200_stream_style& s, uint32_t fields) {
    glava_b200_stream_style k;
    memset(&k, 0, sizeof(k));
    k.set = s.set & fields;
    if (k.set & GLAVA_B200_STYLE_AMPLIFY) k.amplify = s.amplify;
    if (k.set & GLAVA_B200_STYLE_FG) {
        k.fg.mode = s.fg.mode;
        memcpy(k.fg.lo, s.fg.lo, sizeof(k.fg.lo));
        if (s.fg.mode != 1) { memcpy(k.fg.hi, s.fg.hi, sizeof(k.fg.hi)); k.fg.gradient = s.fg.gradient; }
    }
    if (k.set & GLAVA_B200_STYLE_BG) memcpy(k.bg, s.bg, sizeof(k.bg));
    return k;
}
static int style_find(const std::vector<glava_b200_stream_style>& keys, const glava_b200_stream_style& k) {
    for (size_t i = 0; i < keys.size(); ++i) if (!memcmp(&keys[i], &k, sizeof(k))) return (int) i;
    return -1;
}

extern "C" int glava_b200_parse_hex_color(const char* text, float rgba[4]) {
    clear_error();
    if (!text || !rgba) return fail(GLAVA_B200_EINVAL, "glava_b200_parse_hex_color: null argument");
    float c[4];
    if (text[0] != '#' || !parse_hex_color(text, c, true)) return fail(GLAVA_B200_EINVAL, "'%s' is not a #rrggbb[aa] colour", text);
    memcpy(rgba, c, sizeof(c));
    return 0;
}

extern "C" int glava_b200_style_params(const glava_b200_params* base, const glava_b200_stream_style* s, glava_b200_params* out) {
    clear_error();
    if (!base || !s || !out) return fail(GLAVA_B200_EINVAL, "glava_b200_style_params: null argument");
    return style_apply(*base, *s, out);
}

// Everything derived from the parameters that does not depend on the audio (ConfigTables), built into `tb` for the
// parameters of `d` and the stream styles `styles` ([batch], or empty).  Its kernels run on the handle's stream.
static int build_tables(glava_b200* r, const Derived& d, const std::vector<glava_b200_stream_style>& styles, ConfigTables& tb) {
    const glava_b200_params& p = d.p;
    cudaStream_t st = r->stream;
    int rc;
    SpectrumDevTables& sd = tb.spec;
    if (p.transform_smooth) {
        // transform_smooth's sampling window of output t (render.c:700-707) depends on t and the parameters only:
        // evaluated once on the host (chain_core.h), with the same libm calls and types as the reference
        const int sz = p.n;
        std::vector<SmoothWin> win;
        tb.ts_asz = transform_smooth_windows(sz, p.smooth_distance, p.smooth_ratio, &win, &tb.ts_lim);
        if ((rc = table_buf(tb, &tb.ts_tab, (size_t) sz * sizeof(SmoothWin), st, win.data())) != 0) return rc;
    }
    int sm_count = 0;
    if (cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, r->device) != cudaSuccess || sm_count <= 0) {
        cudaGetLastError(); sm_count = 132;                        // H100 SXM
    }
    SpectrumTables host;
    const SpectrumKnobs knobs = spectrum_knobs([](const char* name) -> const char* { return getenv(name); });
    tb.plan = plan_spectrum(p, d.post_chain, r->batch, sm_count, knobs, &host);
    const SpectrumPlan& pl = tb.plan;
    const LazyTables& lt = host.lazy;
    if (pl.need_list) {
        if ((rc = table_buf(tb, &sd.need, lt.need.size() * sizeof(int), st, lt.need.data())) != 0) return rc;
        sd.need_count = (int) lt.cnt;
    }
    if (pl.tap_table) {
        // tap-major for the L2 path, texel-major blob per channel for the shared-memory path and the need-list kernels
        if ((rc = table_buf(tb, &sd.tap_tab, lt.tab.size() * sizeof(TapEntry), st, lt.tab.data())) != 0 ||
            (rc = table_buf(tb, &sd.tap_cnt, lt.tcnt.size() * sizeof(int), st, lt.tcnt.data())) != 0 ||
            (rc = table_buf(tb, &sd.tap_wsum, lt.wsum.size() * sizeof(float), st, lt.wsum.data())) != 0 ||
            (rc = table_buf(tb, &sd.csr, lt.csr.size(), st, lt.csr.data())) != 0) return rc;
        sd.tap_max = (int) lt.tap_max;
        sd.csr_bytes = (int) lt.blob; sd.csr_idx_off = (int) lt.idx_off; sd.csr_off_off = (int) lt.off_off;
    }
    if (pl.k5 == K5Form::NEED_SMEM) {
        const NeedBlocks& nb = host.blocks;
        if ((rc = table_buf(tb, &sd.need_blk, nb.blk.size() * sizeof(int), st, nb.blk.data())) != 0) return rc;
        sd.need_nblk = nb.nblk; sd.need_max_rows = nb.max_rows;
    } else if (pl.k5 == K5Form::NEED_L2) {
        if ((rc = table_buf(tb, &sd.av_t, (size_t) 2 * pl.av_t_len * r->batch * sizeof(float), st, nullptr, true)) != 0) return rc;
    }
    if (pl.full_table) {
        // the taps of ALL n output texels (tables.h build_k5_table_host) for k5_table_kernel
        static_assert(sizeof(K5Blk) == sizeof(int4) && sizeof(K5Ent) == sizeof(int2), "table records are read as int4 / int2");
        const K5TableHost& kt = host.full;
        if ((rc = table_buf(tb, &sd.k5.blk, kt.blk.size() * sizeof(K5Blk), st, kt.blk.data())) != 0 ||
            (rc = table_buf(tb, &sd.k5.ent, kt.ent.size() * sizeof(K5Ent), st, kt.ent.data())) != 0 ||
            (rc = table_buf(tb, &sd.k5.wsum, kt.wsum.size() * sizeof(float), st, kt.wsum.data())) != 0) return rc;
        sd.k5.out = nullptr; sd.k5.count = (int) kt.out.size(); sd.k5.max_span = kt.max_span;
        sd.k5.smem_bytes = K5_S_PLANES * kt.max_span * (int) sizeof(float);
    }
    // Style slots: slot 0 is the renderer's own look, every distinct style of `styles` one more slot (sp: its effective
    // parameters); radial keeps a geometry cache per distinct (fg, bg) pair of the slots (geo_of)
    std::vector<glava_b200_params> sp(1, p);
    std::vector<int> slot_of, geo_of(1, 0);
    if (!styles.empty()) {
        const uint32_t colours = GLAVA_B200_STYLE_FG | GLAVA_B200_STYLE_BG;
        std::vector<glava_b200_stream_style> keys(1, style_key(styles[0], 0)), pairs(1, style_key(styles[0], 0));
        slot_of.assign((size_t) r->batch, 0);
        for (int s = 0; s < r->batch; ++s) {
            const glava_b200_stream_style k = style_key(styles[(size_t) s], ~0u);
            int slot = style_find(keys, k);
            if (slot < 0) {
                glava_b200_params q;
                if ((rc = style_fields(p, k, &q)) != 0) return rc;
                const glava_b200_stream_style pk = style_key(k, colours);
                int g = style_find(pairs, pk);
                if (g < 0) { g = (int) pairs.size(); pairs.push_back(pk); }
                slot = (int) keys.size(); keys.push_back(k); sp.push_back(q); geo_of.push_back(g);
            }
            slot_of[(size_t) s] = slot;
        }
    }
    const int nslots = (int) sp.size();
    int ngeo = 0;
    for (int g : geo_of) ngeo = g + 1 > ngeo ? g + 1 : ngeo;
    const glava_b200_params reach = style_reach_params(p, sp.data(), nslots);
    const RasterTables rt = raster_tables(reach, raster_knobs([](const char* name) -> const char* { return getenv(name); }), nslots, ngeo);
    const bool rows = p.module == GLAVA_B200_MOD_BARS || p.module == GLAVA_B200_MOD_GRAPH;
    if ((rc = table_buf(tb, &tb.rowtab, (size_t) nslots * p.h * 8, st, nullptr, true)) != 0) return rc;
    for (int k = 0; rows && k < nslots; ++k) {
        if ((rc = launch_bars_rowtab(sp[(size_t) k], (char*) tb.rowtab + (size_t) k * p.h * 8, st)) != 0) return rc;
        ++r->launches;
    }
    // polar modules: the audio-independent per-pixel geometry (radial: of every (fg, bg) pair, in the slots' common box)
    if (rt.geo) {
        if ((rc = table_buf(tb, &tb.geo, rt.geo_bytes * rt.geo_caches, st, nullptr)) != 0) return rc;
        for (int g = 0; g < rt.geo_caches; ++g) {
            int k = 0;
            while (geo_of[(size_t) k] != g) ++k;
            if ((rc = launch_polar_geo(sp[(size_t) k], (char*) tb.geo + (size_t) g * rt.geo_bytes, rt.box, st)) != 0) return rc;
            ++r->launches;
        }
    }
    if (nslots > 1) {
        std::vector<StyleSlot> rec((size_t) nslots);
        for (int k = 0; k < nslots; ++k) {
            rec[(size_t) k].p = raster_view(sp[(size_t) k]);
            rec[(size_t) k].rowtab = (const char*) tb.rowtab + (size_t) k * p.h * 8;
            rec[(size_t) k].geo = !rt.geo ? nullptr
                                : (const char*) tb.geo + (p.module == GLAVA_B200_MOD_RADIAL ? (size_t) geo_of[(size_t) k] * rt.geo_bytes : 0);
        }
        StyleSlot* d_rec = nullptr; int* d_of = nullptr;
        if ((rc = table_buf(tb, &d_rec, rec.size() * sizeof(StyleSlot), st, rec.data())) != 0 ||
            (rc = table_buf(tb, &d_of, slot_of.size() * sizeof(int), st, slot_of.data())) != 0) return rc;
        tb.styles = d_rec; tb.style_of = d_of;
        // the host copies of `rec` and `slot_of` must outlive the uploads
        CU(cudaStreamSynchronize(st));
    }
    if (rt.ctile) {
        int ntx = 0, nty = 0;
        const size_t tile_bytes = circle_tile_bytes(p, &ntx, &nty);
        if ((rc = table_buf(tb, &tb.ctile, tile_bytes, st, nullptr)) != 0) return rc;
        if ((rc = launch_circle_tiles(p, tb.geo, rt.box, tb.ctile, st)) != 0) return rc;
        tb.ctile_nx = ntx; tb.ctile_count = ntx * nty;
        r->launches += 2;
    }
    tb.raster = rt;
    CU(cudaStreamSynchronize(st));
    return 0;
}

static int alloc_frame_buffers(glava_b200* r, const glava_b200_params& p, FrameBuffers& f) {
    int rc;
    if ((p.module == GLAVA_B200_MOD_GRAPH || p.module == GLAVA_B200_MOD_WAVE) &&
        (rc = alloc_zeroed(f.coltab, (size_t) r->batch * GLB_COLTAB_PLANES * p.w * sizeof(float), r->stream)) != 0) return rc;
    if ((rc = alloc_zeroed(f.fb, (size_t) p.w * p.h * 4 * r->slots, r->stream)) != 0) return rc;
    return alloc_zeroed(f.marks, mark_bytes(p, r->slots), r->stream);    // empty marks: the framebuffer starts all 0
}

static int sync_all(glava_b200* r) {
    CU(cudaStreamSynchronize(r->spec_stream));
    CU(cudaStreamSynchronize(r->stream));
    if (r->out_stream.get()) CU(cudaStreamSynchronize(r->out_stream));
    return 0;
}

// The one path that builds the renderer for the user parameters `q`: at creation, on glava_b200_reconfigure and on a resize.
// It releases what the new parameters replace first — the tables, and the frame buffers when the geometry changes or they
// are missing — so that a rebuild never holds two sets at once, then builds, and commits parameters, flags, tables and
// plan together once everything has succeeded.  On failure the renderer is unbuilt: it holds no tables, keeps the
// parameters of its last successful build, and refuses to run (frame_ready) until a rebuild succeeds.
static int rebuild(glava_b200* r, const glava_b200_params& q, const std::vector<glava_b200_stream_style>& styles) {
    int rc = validate_params(&q);
    if (rc) return rc;
    // every style must suit the new parameters (style_params of them is what its stream renders)
    std::vector<glava_b200_stream_style> seen;
    for (const glava_b200_stream_style& s : styles) {
        const glava_b200_stream_style k = style_key(s, ~0u);
        if (!k.set || style_find(seen, k) >= 0) continue;
        glava_b200_params tmp;
        if ((rc = style_apply(q, s, &tmp)) != 0) return rc;
        seen.push_back(k);
    }
    const Derived d = derive(q);
    if ((rc = sync_all(r)) != 0) return rc;
    const bool new_frame = !r->built || !r->frame.fb.get() || q.w != r->d.user.w || q.h != r->d.user.h;
    r->built = false;
    r->tab = ConfigTables();
    if (new_frame) r->frame = FrameBuffers();
    FrameBuffers f;
    ConfigTables tb;
    if (new_frame && (rc = alloc_frame_buffers(r, d.p, f)) != 0) return rc;
    if ((rc = build_tables(r, d, styles, tb)) != 0) return rc;
    r->d = d;
    r->tab = std::move(tb);
    if (new_frame) { r->frame = std::move(f); r->mark_key = 0; }
    r->built = true;
    return 0;
}

// The per-stream state, inputs and constants for the parameters of `d`, sized by parameters that never change on a live renderer
static int build_state(glava_b200* r, const Derived& d) {
    const glava_b200_params& p = d.p;
    const size_t n = (size_t) p.n, planes = (size_t) r->batch * 2, F = (size_t) p.avg_frames;
    CU(cudaSetDevice(r->device));
    int rc;
    if ((rc = r->stream.create(0)) != 0) return rc;
    {
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        // Spectrum stream priority: lowest, so that the spectrum kernel of update i+1 fills what the raster kernel of
        // update i leaves free instead of taking each SM's registers first (H100 SXM, 400 W, bars 1080p x 1024 streams:
        // lowest and equal within 0.1 %, high 1 % slower).  GLAVA_B200_SPEC_PRIO=high|equal overrides.
        const char* pr = getenv("GLAVA_B200_SPEC_PRIO");
        int prio = lo;
        if (pr && !strcmp(pr, "high")) prio = hi; else if (pr && !strcmp(pr, "equal")) prio = 0;
        if (getenv("GLAVA_B200_NO_OVERLAP")) r->spec_stream = r->stream;   // tuning aid: serialise spectrum and raster
        else {
            if ((rc = r->own_spec_stream.create(prio)) != 0) return rc;
            r->spec_stream = r->own_spec_stream;
        }
    }
    for (int i = 0; i < 2; ++i)
        if ((rc = r->ev_spec_done[i].create()) != 0 || (rc = r->ev_raster_done[i].create()) != 0) return rc;
    cudaStream_t st = r->stream;
#define ALLOC(buf, bytes) if ((rc = alloc_zeroed((buf), (bytes), st)) != 0) return rc
    if ((rc = r->copy_stream.create(0)) != 0) return rc;
    const size_t n_in = (size_t) d.n_in;
    for (int i = 0; i < 2; ++i) {
        ALLOC(r->d_pcm[i][0], (size_t) r->batch * n_in * 4); ALLOC(r->d_pcm[i][1], (size_t) r->batch * n_in * 4);
        if ((rc = r->ev_copied[i].create()) != 0 || (rc = r->ev_free[i].create()) != 0) return rc;
    }
    for (int i = 0; i < 2; ++i) for (int c = 0; c < 2; ++c) ALLOC(r->d_ring[i][c], (size_t) r->batch * n_in * 4);
    if (d.user.bufscale > 1 || d.user.transform_smooth == 2) { ALLOC(r->d_scaled[0], (size_t) r->batch * n * 4); ALLOC(r->d_scaled[1], (size_t) r->batch * n * 4); }
    if (d.interp_on) {
        for (int i = 0; i < 3; ++i) ALLOC(r->d_key[i], planes * n * 4);      // keyframes start at 0 (render.c:1681 calloc)
        r->key_start = 0; r->key_end = 1;
    }
    if ((rc = r->d_window.alloc(n * 8)) != 0 || (rc = r->d_twiddle.alloc(n * 4)) != 0) return rc;
    ALLOC(r->d_spec, planes * n * 4);
    r->d_spec_cur = r->d_spec;
    // gravity + average state: ONE allocation, so a single L2 access-policy window can cover it (below)
    size_t state_bytes = 0;
    if (p.accel_fft) {
        state_bytes = planes * n * 2 * (1 + F);
        ALLOC(r->d_state, state_bytes);
        r->d_gr_store = (uint16_t*) r->d_state.get(); r->d_ring_u = (uint16_t*) ((char*) r->d_state + planes * n * 2);
    } else {
        state_bytes = planes * n * 4 * (1 + F);
        ALLOC(r->d_state, state_bytes);
        r->d_applied = (float*) r->d_state.get(); r->d_ring_f = (float*) ((char*) r->d_state + planes * n * 4);
    }
    // EXPERIMENT, off by default (GLAVA_B200_L2_PERSIST=1): pin the spectrum kernel's read-modify-write
    // state in the 50 MB L2 with a persisting access window, so that its DRAM reads do not get mixed into
    // the raster kernel's write stream.  Off because the persisting carve-out takes L2 away from the raster
    // kernel's write-back path.
    if (getenv("GLAVA_B200_L2_PERSIST")) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, r->device) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
            size_t want = state_bytes < (size_t) prop.persistingL2CacheMaxSize ? state_bytes : (size_t) prop.persistingL2CacheMaxSize;
            cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want);
            cudaStreamAttrValue attr;
            memset(&attr, 0, sizeof(attr));
            size_t win = state_bytes < (size_t) prop.accessPolicyMaxWindowSize ? state_bytes : (size_t) prop.accessPolicyMaxWindowSize;
            attr.accessPolicyWindow.base_ptr = r->d_state;
            attr.accessPolicyWindow.num_bytes = win;
            attr.accessPolicyWindow.hitRatio = win > 0 ? (float) ((double) want / (double) win) : 0.0f;
            if (attr.accessPolicyWindow.hitRatio > 1.0f) attr.accessPolicyWindow.hitRatio = 1.0f;
            attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
            attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
            if (cudaStreamSetAttribute(r->spec_stream, cudaStreamAttributeAccessPolicyWindow, &attr) != cudaSuccess) cudaGetLastError();
        }
    }
    ALLOC(r->d_tex, 2 * planes * n * 2);
    ALLOC(r->d_av, planes * n * 2);
    ALLOC(r->d_texmm, planes * GLB_TEXMM_STRIDE * sizeof(uint32_t));          // one buffer: texmm_kernel fills it on the raster stream right before the circle raster reads it
#undef ALLOC
    r->slots = (p.fb_slots > 0 && p.fb_slots < r->batch) ? p.fb_slots : r->batch;
    // window LUT: render.c:660 macro as expanded at render.c:794 — cos(TWOPI*i/N - 1), double
    std::vector<double> w(n);
    for (size_t i = 0; i < n; ++i) w[i] = 0.53836 - (0.46164 * cos(6.28318530718 * (double) i / (double) n - 1));
    CU(cudaMemcpyAsync(r->d_window, w.data(), n * 8, cudaMemcpyHostToDevice, st));
    // twiddles exp(-2*pi*i*k/M), M = n/2, evaluated in double
    const size_t M = n / 2;
    std::vector<float> tw(2 * M);
    for (size_t k = 0; k < M; ++k) {
        double ang = -2.0 * M_PI * (double) k / (double) M;
        tw[2 * k] = (float) cos(ang); tw[2 * k + 1] = (float) sin(ang);
    }
    CU(cudaMemcpyAsync(r->d_twiddle, tw.data(), n * 4, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    return 0;
}

glava_b200* glava_b200_new(const glava_b200_params* params, int batch, int device) {
    clear_error();
    if (!params || batch < 1) { fail(GLAVA_B200_EINVAL, "glava_b200_new: bad arguments"); return nullptr; }
    if (validate_params(params) != 0) return nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        fail(GLAVA_B200_ECUDA, "no CUDA device available: the GPU path has no CPU fallback");
        return nullptr;
    }
    if (device < 0 || device >= ndev) { fail(GLAVA_B200_EINVAL, "device %d out of range (%d devices)", device, ndev); return nullptr; }
    glava_b200* r = new glava_b200();
    r->batch = batch; r->device = device;
    if (build_state(r, derive(*params)) != 0 || rebuild(r, *params, r->styles) != 0) { glava_b200_destroy(r); return nullptr; }
    return r;
}

void glava_b200_destroy(glava_b200* r) {
    if (!r) return;
    cudaSetDevice(r->device);
    for (cudaStream_t s : { r->spec_stream, r->stream.get(), r->copy_stream.get(), r->out_stream.get() })
        if (s) cudaStreamSynchronize(s);
    if (r->attach_free) r->attach_free(r->attach);
    delete r;
}

int glava_b200_reconfigure(glava_b200* r, const glava_b200_params* params) {
    clear_error();
    if (!r || !params) return fail(GLAVA_B200_EINVAL, "glava_b200_reconfigure: null argument");
    int rc = validate_params(params);
    if (rc) return rc;
    const glava_b200_params& o = r->d.user;
    if (params->n != o.n || params->w != o.w || params->h != o.h || params->module != o.module || params->accel_fft != o.accel_fft ||
        params->avg_frames != o.avg_frames || params->fb_slots != o.fb_slots || params->bufscale != o.bufscale ||
        params->transform_smooth != o.transform_smooth || derive(*params).interp_on != r->d.interp_on)
        return fail(GLAVA_B200_EINVAL, "glava_b200_reconfigure: setbufsize, setbufscale, geometry, module, setaccelfft, setavgframes, "
                                       "fb_slots, the \"smooth\" transform and whether interpolation is active size the device "
                                       "state and cannot change on a live renderer; create a new one");
    CU(cudaSetDevice(r->device));
    return rebuild(r, *params, r->styles);
}

int glava_b200_get_params(const glava_b200* r, glava_b200_params* out) {
    if (!r || !out) return fail(GLAVA_B200_EINVAL, "null argument");
    *out = r->d.user; return 0;
}
int glava_b200_batch(const glava_b200* r) { return r ? r->batch : 0; }
const char* glava_b200_module_name(const glava_b200* r) { return r ? module_name(r->d.p.module) : "?"; }
int glava_b200_spectrum_size(const glava_b200* r) { return r ? r->d.p.n : 0; }
const void* glava_b200_framebuffer_device(const glava_b200* r) { return r ? r->frame.fb.get() : nullptr; }
void* glava_b200_cuda_stream(const glava_b200* r) { return r ? (void*) r->stream : nullptr; }
uint64_t glava_b200_launch_count(const glava_b200* r) { return r ? r->launches : 0; }

static int timing_mark(std::vector<Event>& v, cudaStream_t st) {
    Event e;
    int rc = e.create(cudaEventDefault);
    if (rc) return rc;
    CU(cudaEventRecord(e, st));
    v.push_back(std::move(e));
    return 0;
}

static uint16_t* tex_half(glava_b200* r, int b) { return r->d_tex + (size_t) b * r->batch * 2 * r->d.p.n; }
// Runtime resize (render.c:1811-1830 resizes the stage FBOs when the framebuffer size changed; offscreen consumers ask
// through glava_sizereq, glava.c:263-267), applied at the start of a frame (render.c:1811-1815).  Spectrum state is
// untouched; the framebuffers and every table (row colours, polar geometry cache, lazy-K5 need-list) are rebuilt.  Then a
// renderer that a failed reconfigure or resize left unbuilt refuses to run, before anything is enqueued.
static int unbuilt() {
    return fail(GLAVA_B200_ECUDA, "the renderer has no tables: a reconfigure or resize failed and must be repeated");
}
static int frame_ready(glava_b200* r) {
    if (unsigned long long req = r->sizereq.exchange(0)) {
        glava_b200_params q = r->d.user;
        q.w = (int) ((req >> 32) & 0x7fffffffu); q.h = (int) (req & 0xffffffffu);
        int rc = rebuild(r, q, r->styles);
        if (rc) return rc;
    }
    return r->built ? 0 : unbuilt();
}

// Per-stream mask -> device words.  Returns the device array for this update (nullptr: every stream modified in lock step).
static int stage_umask(glava_b200* r, const uint8_t* mask, const uint32_t** d_out) {
    const int F = r->d.p.avg_frames;
    if (!r->desync) {                                           // first uneven update: every stream starts from the shared cursor
        r->cursor.assign((size_t) r->batch, (uint32_t) (r->updates % (unsigned long long) F));
        r->desync = true;
    }
    const int k = r->umask_cur;
    if (!r->ev_umask[k].get()) {                              // created last: the slot is complete
        int rc;
        if ((rc = r->h_umask[k].alloc((size_t) r->batch * 4)) != 0 || (rc = r->d_umask[k].alloc((size_t) r->batch * 4)) != 0 ||
            (rc = r->ev_umask[k].create()) != 0) return rc;
    } else {
        CU(cudaEventSynchronize(r->ev_umask[k]));               // the copy that last read this pinned buffer (4 updates ago)
    }
    for (int s = 0; s < r->batch; ++s) {
        const bool m = !mask || mask[s];
        r->h_umask[k][s] = (m ? 0x80000000u : 0u) | r->cursor[s];
        if (m) r->cursor[s] = (r->cursor[s] + 1u) % (uint32_t) F;
    }
    CU(cudaMemcpyAsync(r->d_umask[k], r->h_umask[k], (size_t) r->batch * 4, cudaMemcpyHostToDevice, r->spec_stream));
    CU(cudaEventRecord(r->ev_umask[k], r->spec_stream));
    r->umask_cur = (k + 1) & 3;
    *d_out = r->d_umask[k];
    return 0;
}

// One update's input, as a public entry point received it
struct UpdateInput {
    enum Source { HOST, DEVICE, RINGS, TEXTURES } src;
    const char* who;                  // the public function, for error messages
    const void* l = nullptr, *r = nullptr;   // HOST / DEVICE: PCM [batch][bsz]; TEXTURES: R16 [batch][n]; r may be null
    size_t bsz = 0;                   // HOST / DEVICE: floats per stream and channel
    bool modified = false;            // every stream has new audio
    const uint8_t* mask = nullptr;    // or: one byte per stream, non-zero = that stream has new audio (glava.c:528-537 per renderer)
    void* ready = nullptr;            // DEVICE: a cudaEvent_t the PCM is written behind (glava_b200_update_device_after), or null
};

// Everything an update checks before it enqueues anything, in this order.  A mask leaves here normalised: `modified` says
// whether any stream has new audio, and a mask that marks none or all of them gives way to the plain form.
static int check_update(glava_b200* r, UpdateInput& in) {
    const bool pcm = in.src == UpdateInput::HOST || in.src == UpdateInput::DEVICE;
    if (pcm && in.bsz != (size_t) r->d.n_in) return fail(GLAVA_B200_EINVAL, "%s: bsz %zu != setbufsize %d", in.who, in.bsz, r->d.n_in);
    if (in.src == UpdateInput::DEVICE && (((uintptr_t) in.l & 15) || ((uintptr_t) in.r & 15)))
        return fail(GLAVA_B200_EINVAL, "device PCM pointers must be 16-byte aligned");
    int cnt = 0;
    for (int s = 0; in.mask && s < r->batch; ++s) cnt += in.mask[s] ? 1 : 0;
    if (in.mask) in.modified = cnt > 0;
    // rd_update always gets both rings (render.h:58); only `wave` ignores rb (wave/1.frag:7 samples audio_l alone).  A masked
    // update from device pointers asks for d_rb whatever its mask.
    if (pcm && !in.r && r->d.p.module != GLAVA_B200_MOD_WAVE && (in.modified || (in.mask && in.src == UpdateInput::DEVICE)))
        return fail(GLAVA_B200_EINVAL, "%s: module '%s' reads both channels, %s is null", in.who, module_name(r->d.p.module),
                    in.src == UpdateInput::HOST ? "rb" : "d_rb");
    CU(cudaSetDevice(r->device));
    int rc;
    if (in.src == UpdateInput::HOST && (rc = frame_ready(r)) != 0) return rc;     // host input: before the mask
    if (in.mask && (cnt == 0 || cnt == r->batch)) in.mask = nullptr;               // nobody / everybody: the plain forms
    if (in.mask && r->d.interp_on)
        return fail(GLAVA_B200_EINVAL, "per-stream modified masks are not available with keyframe interpolation active "
                                       "(setinterpolate): the keyframe rotation is per renderer; update the streams in lock step");
    if (in.src != UpdateInput::HOST && (rc = frame_ready(r)) != 0) return rc;
    // a K5 form the plan refuses (spectrum_plan.h) fails every update with a new texture
    const bool new_tex = in.src != UpdateInput::TEXTURES && (in.modified || r->d.interp_on);
    if (new_tex && !r->tab.plan.refusal.empty()) return fail(GLAVA_B200_EINVAL, "%s", r->tab.plan.refusal.c_str());
    return 0;
}

// The keyframe buffer that is neither the start nor the end of the interpolation: the next update's chain result goes there
static int next_key(const glava_b200* r) { int k = 0; while (k == r->key_start || k == r->key_end) ++k; return k; }

// The spectrum half of an update, on spec_stream, from device PCM [batch][n_in]: the stages in front of the FFT, the spectrum
// update in the launch structure build_tables chose (spectrum_plan.h), the post chain and the keyframe rotation
static int enqueue_spectrum(glava_b200* r, const float* d_l, const float* d_r, bool modified, const uint8_t* mask) {
    const glava_b200_params& p = r->d.p;
    const bool new_tex = modified || r->d.interp_on;      // an interpolated frame has a new texture without new audio
    const int planes = r->batch * 2;
    const size_t total = (size_t) planes * p.n;
    int rc;
    if (new_tex) CU(cudaStreamWaitEvent(r->spec_stream, r->ev_raster_done[r->tex_cur ^ 1], 0));
    if (modified && r->d.user.bufscale > 1) {
        const int chans = p.module == GLAVA_B200_MOD_WAVE ? 1 : 2;
        if ((rc = launch_bufscale(d_l, d_r, r->d_scaled[0], r->d_scaled[1], r->batch, r->d.n_in, r->d.user.bufscale, chans, r->spec_stream)) != 0) return rc;
        ++r->launches;
        d_l = r->d_scaled[0]; d_r = r->d_scaled[1];
    }
    if (modified && p.transform_smooth == 2) {
        // `#request transform <u> "smooth"` listed BEFORE "fft" (render.c:1218-1286): handle_audio applies it on the CPU to
        // the (scaled) PCM ring, then meets "fft" and carries on as usual (render.c:2131-2156).  Here: on a copy of the
        // rings (rd_update transforms the caller's buffers in place; this ABI leaves them alone)
        const int chans = p.module == GLAVA_B200_MOD_WAVE ? 1 : 2;
        const float* src[2] = { d_l, d_r };
        for (int c = 0; c < chans; ++c) {
            if (src[c] != r->d_scaled[c]) CU(cudaMemcpyAsync(r->d_scaled[c], src[c], (size_t) r->batch * p.n * 4, cudaMemcpyDeviceToDevice, r->spec_stream));
            if ((rc = launch_transform_smooth(r->d_scaled[c], p.n, r->tab.ts_tab, r->tab.ts_asz, r->tab.ts_lim, r->batch, r->spec_stream, nullptr, 0)) != 0) return rc;
            ++r->launches;
        }
        d_l = r->d_scaled[0]; d_r = chans == 2 ? r->d_scaled[1] : r->d_scaled[0];
    }
    float* chain_out = r->d_spec;                         // where the float chain result of this update goes
    if (r->d.interp_on) chain_out = r->d_key[next_key(r)];
    if (modified) {
        const int b = r->tex_cur ^ 1;
        SpectrumArgs a = r->d.spec_args;
        a.pcm_l = d_l; a.pcm_r = d_r; a.window = r->d_window; a.twiddle = r->d_twiddle;
        a.spec = chain_out; a.skip_tex = r->d.post_chain ? 1 : 0; a.applied = r->d_applied; a.ring_f = r->d_ring_f;
        a.gr_store = r->d_gr_store; a.ring_u = r->d_ring_u; a.tex = tex_half(r, b); a.av_out = r->d_av;
        a.batch = r->batch; a.update = r->updates;
        a.umask = nullptr; a.tex_prev = tex_half(r, r->tex_cur);
        if (mask || r->desync) { if ((rc = stage_umask(r, mask, &a.umask)) != 0) return rc; }
        if (r->timing && (rc = timing_mark(r->ev_spec, r->spec_stream)) != 0) return rc;
        if ((rc = launch_spectrum_update(p, r->tab.plan, r->tab.spec, a, r->spec_stream)) < 0) return rc;
        r->launches += (uint64_t) rc;
        if (r->d.post_chain && p.transform_smooth == 1) {                     // render.c:694-718, after the module's chain
            if ((rc = launch_transform_smooth(chain_out, p.n, r->tab.ts_tab, r->tab.ts_asz, r->tab.ts_lim, planes, r->spec_stream, a.umask)) != 0) return rc;
            ++r->launches;
        }
        if (!r->d.post_chain) {
            if (r->timing && (rc = timing_mark(r->ev_spec, r->spec_stream)) != 0) return rc;
            CU(cudaEventRecord(r->ev_spec_done[b], r->spec_stream));
            r->tex_cur = b;
        }
        ++r->updates;
        r->d_spec_cur = chain_out;
    }
    if (r->d.post_chain && new_tex) {
        // R16 upload of the buffer this frame shows (render.c:2185) and K5 (render.c:2276-2303).  With keyframe
        // interpolation that is the lerp of the two PREVIOUS post-transform buffers (render.c:1792-1809): the
        // update just computed becomes visible one update later (rc.glsl:129-130).
        const int b = r->tex_cur ^ 1;
        uint16_t* dst = p.smooth_pass ? r->d_av : tex_half(r, b);
        if (r->d.interp_on) {
            const float mod = keyframe_mod(p.ur, p.fr > 0.0f ? p.fr : p.ur, r->kcounter);   // render.c:1761,1804
            rc = launch_upload(r->d_key[r->key_start], r->d_key[r->key_end], mod, dst, total, r->spec_stream);
        } else {
            rc = launch_upload(chain_out, nullptr, 0.0f, dst, total, r->spec_stream);
        }
        if (rc) return rc;
        ++r->launches;
        if (p.smooth_pass) {
            if ((rc = launch_k5_full(p, r->tab.plan, r->tab.spec.k5, r->d_av, tex_half(r, b), planes, r->spec_stream)) != 0) return rc;
            ++r->launches;
        }
        if (modified && r->timing && (rc = timing_mark(r->ev_spec, r->spec_stream)) != 0) return rc;
        CU(cudaEventRecord(r->ev_spec_done[b], r->spec_stream));
        r->tex_cur = b;
        if (r->d.interp_on && modified) {                                       // render.c:2347-2353: start <- end <- this update
            const int nxt = next_key(r);
            r->key_start = r->key_end; r->key_end = nxt;
        }
    }
    r->kcounter = modified ? 0 : r->kcounter + 1;                             // render.c:2380-2383
    return 0;
}

// The raster half of an update, on stream: the raster pass of raster_plan.h (knobs read at every pass) over the latest texture
static int enqueue_raster(glava_b200* r) {
    const int b = r->tex_cur;
    int rc;
    CU(cudaStreamWaitEvent(r->stream, r->ev_spec_done[b], 0));
    const RasterKnobs knobs = raster_knobs([](const char* name) -> const char* { return getenv(name); });
    const glava_b200_params view = raster_view(r->d.p);
    const ConfigTables& tb = r->tab;
    const RasterPlan pl = plan_raster(view, tb.raster, r->batch, r->slots, knobs);
    RasterPass ra = {};
    ra.tex = tex_half(r, b); ra.fb = r->frame.fb;
    ra.rowtab = pl.rowtab ? tb.rowtab : nullptr;
    ra.batch = r->batch; ra.slots = r->slots; ra.stream0 = 0;
    ra.geo = pl.geo ? tb.geo : nullptr;
    ra.gx0 = tb.raster.box[0]; ra.gy0 = tb.raster.box[1]; ra.gw = tb.raster.box[2]; ra.gh = tb.raster.box[3];
    ra.texmm = pl.texmm ? (const uint32_t*) r->d_texmm : nullptr;
    ra.ctile = pl.ctile ? (const int4*) tb.ctile : nullptr;
    ra.ctile_zero = pl.ctile ? (const int*) ((const int4*) tb.ctile + tb.ctile_count) : nullptr;
    ra.ctile_nx = pl.ctile ? tb.ctile_nx : 0;
    ra.coltab = pl.coltab ? (float*) r->frame.coltab : nullptr;
    ra.marks = r->frame.marks; ra.marks_valid = raster_marks_valid(pl, r->mark_key, knobs) ? 1 : 0;
    if (pl.styled) { ra.styles.style_of = tb.style_of; ra.styles.styles = tb.styles; }
    if (pl.texmm && (rc = launch_texmm(r->d.p, ra.tex, r->d_texmm, r->batch * 2, r->stream)) != 0) return rc;
    r->mark_key = 0;                                      // until every launch of the pass is enqueued
    if (r->timing && (rc = timing_mark(r->ev_ras, r->stream)) != 0) return rc;
    if ((rc = launch_raster(view, pl, ra, r->stream)) != 0) return rc;
    r->mark_key = pl.mark_key;
    if (r->timing && (rc = timing_mark(r->ev_ras, r->stream)) != 0) return rc;
    CU(cudaEventRecord(r->ev_raster_done[b], r->stream));
    r->launches += (uint64_t) pl.launches;
    return 0;
}

// One update = the spectrum half on spec_stream (when there is a new texture) + the raster half on stream.
//   spectrum(i) waits for: its input (caller-provided event on spec_stream), spectrum(i-1) (same stream:
//                          gravity / average state is read-modify-write), raster(i-2) (last reader of the
//                          texture half it overwrites)
//   raster(i)   waits for: spectrum(i)
// so raster(i) and spectrum(i+1) run concurrently: one is HBM-store bound, the other latency bound.
static int run_update(glava_b200* r, UpdateInput in) {
    int rc = check_update(r, in);
    if (rc) return rc;
    const float* d_l = (const float*) in.l;
    const float* d_r = in.r ? (const float*) in.r : d_l;
    const int b = r->stage_cur;
    const bool staged = in.src == UpdateInput::HOST && in.modified;
    if (staged) {
        // into staging buffer b once the kernels that last read it are done; on copy_stream, under the previous update
        const size_t bytes = (size_t) r->batch * in.bsz * 4;
        CU(cudaStreamWaitEvent(r->copy_stream, r->ev_free[b], 0));
        CU(cudaMemcpyAsync(r->d_pcm[b][0], in.l, bytes, cudaMemcpyHostToDevice, r->copy_stream));
        if (r->d.p.module != GLAVA_B200_MOD_WAVE) CU(cudaMemcpyAsync(r->d_pcm[b][1], in.r, bytes, cudaMemcpyHostToDevice, r->copy_stream));
        CU(cudaEventRecord(r->ev_copied[b], r->copy_stream));
        CU(cudaStreamWaitEvent(r->spec_stream, r->ev_copied[b], 0));
    }
    if (in.src == UpdateInput::HOST) { d_l = r->d_pcm[b][0]; d_r = r->d_pcm[b][1]; }
    if (in.src == UpdateInput::RINGS) { d_l = r->d_ring[r->ring_cur][0]; d_r = r->d_ring[r->ring_cur][1]; }
    if (in.ready) CU(cudaStreamWaitEvent(r->spec_stream, (cudaEvent_t) in.ready, 0));
    if ((rc = enqueue_spectrum(r, d_l, d_r, in.modified, in.mask)) != 0 || (rc = enqueue_raster(r)) != 0) return rc;
    if (staged) {
        // like rd_update, return once lb / rb are consumed (unless glava_b200_set_async_input)
        CU(cudaEventRecord(r->ev_free[b], r->spec_stream));
        r->stage_cur = b ^ 1;
        r->last_in = b;
        if (!r->async_input) CU(cudaEventSynchronize(r->ev_copied[b]));
    }
    return 0;
}

int glava_b200_update(glava_b200* r, const float* lb, const float* rb, size_t bsz, int modified) {
    clear_error();
    if (!r || !lb) return fail(GLAVA_B200_EINVAL, "glava_b200_update: null argument");
    return run_update(r, { UpdateInput::HOST, "glava_b200_update", lb, rb, bsz, modified != 0 });
}

// Double-buffer contract for the host rings (instead of rd_update's "consumed on return"): with async input enabled
// glava_b200_update* return as soon as the copy is ENQUEUED; the caller keeps lb / rb untouched until
// glava_b200_wait_input() — in practice it alternates between two sets of rings, and the host never blocks on a copy.
int glava_b200_set_async_input(glava_b200* r, int enable) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    r->async_input = enable != 0;
    return 0;
}
int glava_b200_wait_input(glava_b200* r) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    if (r->last_in < 0) return 0;
    CU(cudaSetDevice(r->device));
    CU(cudaEventSynchronize(r->ev_copied[r->last_in]));
    return 0;
}

int glava_b200_update_masked(glava_b200* r, const float* lb, const float* rb, size_t bsz, const uint8_t* modified) {
    clear_error();
    if (!r || !lb || !modified) return fail(GLAVA_B200_EINVAL, "glava_b200_update_masked: null argument");
    return run_update(r, { UpdateInput::HOST, "glava_b200_update_masked", lb, rb, bsz, true, modified });
}

int glava_b200_update_device_masked(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, const uint8_t* modified) {
    clear_error();
    if (!r || !d_lb || !modified) return fail(GLAVA_B200_EINVAL, "glava_b200_update_device_masked: null argument");
    return run_update(r, { UpdateInput::DEVICE, "glava_b200_update_device_masked", d_lb, d_rb, bsz, true, modified });
}

int glava_b200_update_rings_masked(glava_b200* r, const uint8_t* modified) {
    clear_error();
    if (!r || !modified) return fail(GLAVA_B200_EINVAL, "glava_b200_update_rings_masked: null argument");
    return run_update(r, { UpdateInput::RINGS, "glava_b200_update_rings_masked", nullptr, nullptr, 0, true, modified });
}

// Ordering of glava_b200_update_device against the caller's own CUDA work.  The spectrum kernel reads d_lb / d_rb on an
// internal non-blocking stream: hand over the event that marks "buffers written" (recorded on the producer's stream) and the
// kernel waits for it on the device; glava_b200_input_event() is recorded after the kernel that last READ the buffers, so
// the producer can cudaStreamWaitEvent on it before overwriting them.  Both are cudaEvent_t passed as void*.
int glava_b200_update_device_after(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, int modified, void* ready_event) {
    clear_error();
    if (!r || !d_lb) return fail(GLAVA_B200_EINVAL, "glava_b200_update_device_after: null argument");
    return run_update(r, { UpdateInput::DEVICE, "glava_b200_update_device_after", d_lb, d_rb, bsz, modified != 0, nullptr, ready_event });
}
void* glava_b200_input_event(glava_b200* r) {
    if (!r) return nullptr;
    if (!r->ev_input.get() && r->ev_input.create() != 0) return nullptr;
    cudaSetDevice(r->device);
    cudaEventRecord(r->ev_input, r->spec_stream);          // after everything enqueued so far on the reading stream
    return (void*) r->ev_input;
}

int glava_b200_update_device(glava_b200* r, const float* d_lb, const float* d_rb, size_t bsz, int modified) {
    clear_error();
    if (!r || !d_lb) return fail(GLAVA_B200_EINVAL, "glava_b200_update_device: null argument");
    return run_update(r, { UpdateInput::DEVICE, "glava_b200_update_device", d_lb, d_rb, bsz, modified != 0 });
}

static int ingest(glava_b200* r, const void* chunks, bool float_in, int frames, const char* who) {
    clear_error();
    if (!r || !chunks) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    if (frames < 1 || frames > r->d.n_in) return fail(GLAVA_B200_EINVAL, "%s: frames %d out of range", who, frames);
    CU(cudaSetDevice(r->device));
    size_t bytes = (size_t) r->batch * frames * 2 * (float_in ? sizeof(float) : sizeof(int16_t));
    if (bytes > r->chunks_cap) {
        CU(cudaStreamSynchronize(r->spec_stream));
        r->chunks_cap = 0;
        int rc = r->d_chunks.alloc(bytes);
        if (rc) return rc;
        r->chunks_cap = bytes;
    }
    // ordered with the spectrum kernels (they read the rings): same stream
    CU(cudaMemcpyAsync(r->d_chunks, chunks, bytes, cudaMemcpyHostToDevice, r->spec_stream));
    int cur = r->ring_cur, nxt = cur ^ 1;
    int rc = launch_fifo_ingest(r->d.user, r->d_chunks, float_in, frames, r->d_ring[cur][0], r->d_ring[cur][1],
                                r->d_ring[nxt][0], r->d_ring[nxt][1], r->batch, r->spec_stream);
    if (rc) return rc;
    ++r->launches;
    r->ring_cur = nxt;
    return 0;
}
int glava_b200_ingest_fifo(glava_b200* r, const int16_t* chunks, int frames) { return ingest(r, chunks, false, frames, "glava_b200_ingest_fifo"); }
int glava_b200_ingest_float(glava_b200* r, const float* chunks, int frames) { return ingest(r, chunks, true, frames, "glava_b200_ingest_float"); }

int glava_b200_update_rings(glava_b200* r, int modified) {
    clear_error();
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    return run_update(r, { UpdateInput::RINGS, "glava_b200_update_rings", nullptr, nullptr, 0, modified != 0 });
}

// ---- offscreen hand-off (glava.h:16-25, glava.c:244-267) -----------------------------------------------------------
int glava_b200_sizereq(glava_b200* r, int w, int h) {
    if (!r || w < 1 || h < 1 || w > 0x7fffffff) return fail(GLAVA_B200_EINVAL, "glava_b200_sizereq: bad arguments");
    r->sizereq.store((1ull << 63) | ((unsigned long long) (unsigned) w << 32) | (unsigned) h);
    return 0;
}
int glava_b200_wait_frame(glava_b200* r) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    CU(cudaEventSynchronize(r->ev_raster_done[r->tex_cur]));
    return 0;
}
void* glava_b200_frame_event(const glava_b200* r) { return r ? (void*) r->ev_raster_done[r->tex_cur] : nullptr; }
const void* glava_b200_frame_device(const glava_b200* r, int stream) {
    if (!r || stream < 0 || stream >= r->batch || !r->frame.fb) return nullptr;
    return r->frame.fb + (size_t) r->d.p.w * r->d.p.h * 4 * (size_t) (stream % r->slots);
}
int glava_b200_framebuffer_ipc(glava_b200* r, void* handle, size_t handle_bytes) {
    clear_error();
    if (!r || !handle || handle_bytes < sizeof(cudaIpcMemHandle_t)) return fail(GLAVA_B200_EINVAL, "glava_b200_framebuffer_ipc: need a %zu-byte buffer", sizeof(cudaIpcMemHandle_t));
    CU(cudaSetDevice(r->device));
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, r->frame.fb));
    memcpy(handle, &h, sizeof(h));
    return 0;
}

int glava_b200_set_timing(glava_b200* r, int enable) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    int rc0 = sync_all(r); if (rc0) return rc0;
    r->ev_spec.clear(); r->ev_ras.clear();
    r->timing = enable != 0;
    return 0;
}

int glava_b200_kernel_times(glava_b200* r, double* spectrum_ms, int* spectrum_launches, double* raster_ms, int* raster_launches) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    int rc0 = sync_all(r); if (rc0) return rc0;
    double s = 0, q = 0; int ns = 0, nq = 0;
    for (size_t i = 0; i + 1 < r->ev_spec.size(); i += 2) {
        float a = 0; CU(cudaEventElapsedTime(&a, r->ev_spec[i], r->ev_spec[i + 1])); s += a; ++ns;
    }
    for (size_t i = 0; i + 1 < r->ev_ras.size(); i += 2) {
        float a = 0; CU(cudaEventElapsedTime(&a, r->ev_ras[i], r->ev_ras[i + 1])); q += a; ++nq;
    }
    if (spectrum_ms) *spectrum_ms = s;
    if (spectrum_launches) *spectrum_launches = ns;
    if (raster_ms) *raster_ms = q;
    if (raster_launches) *raster_launches = nq;
    return 0;
}

// Event timeline of the timed launches, in ms relative to the first spectrum mark: out = [start, end] pairs, spectrum
// launches first (n_spec pairs) then raster launches.  Development aid for looking at the overlap of the two streams.
int glava_b200_timeline(glava_b200* r, double* out, int cap_pairs, int* n_spec, int* n_ras) {
    if (!r || !out) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    int rc0 = sync_all(r); if (rc0) return rc0;
    const int ns = (int) r->ev_spec.size() / 2, nq = (int) r->ev_ras.size() / 2;
    if (ns + nq > cap_pairs || ns == 0) return fail(GLAVA_B200_EINVAL, "glava_b200_timeline: %d pairs, capacity %d", ns + nq, cap_pairs);
    cudaEvent_t t0 = r->ev_spec[0];
    for (int i = 0; i < 2 * ns; ++i) { float a = 0; CU(cudaEventElapsedTime(&a, t0, r->ev_spec[i])); out[i] = a; }
    for (int i = 0; i < 2 * nq; ++i) { float a = 0; CU(cudaEventElapsedTime(&a, t0, r->ev_ras[i])); out[2 * ns + i] = a; }
    if (n_spec) *n_spec = ns;
    if (n_ras) *n_ras = nq;
    return 0;
}

int glava_b200_sync(glava_b200* r) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    return sync_all(r);
}

int glava_b200_readback(glava_b200* r, int stream, uint8_t* rgba) {
    clear_error();
    if (!r || !rgba || stream < 0 || stream >= r->batch) return fail(GLAVA_B200_EINVAL, "glava_b200_readback: bad arguments");
    CU(cudaSetDevice(r->device));
    size_t frame = (size_t) r->d.p.w * r->d.p.h * 4;
    CU(cudaMemcpyAsync(rgba, r->frame.fb + frame * (size_t) (stream % r->slots), frame, cudaMemcpyDeviceToHost, r->stream));
    CU(cudaStreamSynchronize(r->stream));
    return 0;
}

int glava_b200_readback_async(glava_b200* r, int stream, uint8_t* rgba) {
    clear_error();
    if (!r || !rgba || stream < 0 || stream >= r->batch) return fail(GLAVA_B200_EINVAL, "glava_b200_readback_async: bad arguments");
    CU(cudaSetDevice(r->device));
    const size_t frame = (size_t) r->d.p.w * r->d.p.h * 4;
    int rc;
    if (!r->ev_stage_free[1].get()) {                      // created last: the read-back stream and its events are complete
        if ((rc = r->out_stream.create(0)) != 0) return rc;
        for (int i = 0; i < 2; ++i)
            if ((rc = r->ev_stage_ready[i].create()) != 0 || (rc = r->ev_stage_free[i].create()) != 0) return rc;
    }
    if (r->stage_bytes != frame) {                       // first use, or the geometry changed (glava_b200_sizereq)
        CU(cudaStreamSynchronize(r->out_stream));
        r->stage_bytes = 0;
        for (int i = 0; i < 2; ++i) { r->d_stage[i].reset(); }
        for (int i = 0; i < 2; ++i) if ((rc = r->d_stage[i].alloc(frame)) != 0) return rc;
        r->stage_bytes = frame;
    }
    const int i = r->out_cur;
    // the frame is snapshotted on the raster stream (ordered after the raster that produced it, before the next one
    // overwrites the slot); the slow PCIe leg then runs from the snapshot on its own stream
    CU(cudaStreamWaitEvent(r->stream, r->ev_stage_free[i], 0));
    CU(cudaMemcpyAsync(r->d_stage[i], r->frame.fb + frame * (size_t) (stream % r->slots), frame, cudaMemcpyDeviceToDevice, r->stream));
    CU(cudaEventRecord(r->ev_stage_ready[i], r->stream));
    CU(cudaStreamWaitEvent(r->out_stream, r->ev_stage_ready[i], 0));
    CU(cudaMemcpyAsync(rgba, r->d_stage[i], frame, cudaMemcpyDeviceToHost, r->out_stream));
    CU(cudaEventRecord(r->ev_stage_free[i], r->out_stream));
    r->out_cur = i ^ 1;
    return 0;
}

// Orders everything enqueued on the handle's stream from now on after the read-backs issued so far (their PCIe leg runs
// on a separate stream): an event recorded on glava_b200_cuda_stream() after this call covers them.
int glava_b200_readback_fence(glava_b200* r) {
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    if (!r->ev_stage_free[1].get()) return 0;
    CU(cudaSetDevice(r->device));
    for (int i = 0; i < 2; ++i) CU(cudaStreamWaitEvent(r->stream, r->ev_stage_free[i], 0));
    return 0;
}

static int planes_to_host(glava_b200* r, const void* d, size_t elem, void* out_l, void* out_r) {
    // device layout [batch][2][n] -> two host arrays [batch][n]
    const size_t row = (size_t) r->d.p.n * elem;
    CU(cudaStreamSynchronize(r->spec_stream));
    if (out_l) CU(cudaMemcpy2DAsync(out_l, row, d, 2 * row, row, (size_t) r->batch, cudaMemcpyDeviceToHost, r->stream));
    if (out_r) CU(cudaMemcpy2DAsync(out_r, row, (const char*) d + row, 2 * row, row, (size_t) r->batch, cudaMemcpyDeviceToHost, r->stream));
    CU(cudaStreamSynchronize(r->stream));
    return 0;
}
int glava_b200_spectrum(glava_b200* r, float* out_l, float* out_r) {
    clear_error();
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    return planes_to_host(r, r->d_spec_cur, 4, out_l, out_r);
}
int glava_b200_textures(glava_b200* r, uint16_t* out_l, uint16_t* out_r) {
    clear_error();
    if (!r) return fail(GLAVA_B200_EINVAL, "null argument");
    CU(cudaSetDevice(r->device));
    return planes_to_host(r, tex_half(r, r->tex_cur), 2, out_l, out_r);
}

int glava_b200_smooth_pass(glava_b200* r, const uint16_t* in, uint16_t* out, int count) {
    clear_error();
    if (!r || !in || !out || count < 1) return fail(GLAVA_B200_EINVAL, "glava_b200_smooth_pass: bad arguments");
    if (!r->built) return unbuilt();
    CU(cudaSetDevice(r->device));
    // the renderer's whole-plane table when it has one, else k5_planes_kernel where its spans fit shared memory
    const std::string refusal = r->tab.plan.full_table ? std::string() : k5_planes_refusal(k5_planes_span(r->d.p));
    if (!refusal.empty()) return fail(GLAVA_B200_EINVAL, "%s", refusal.c_str());
    const size_t bytes = (size_t) count * r->d.p.n * 2;
    DevBuf<uint16_t> d_in, d_out;
    int rc;
    if ((rc = d_in.alloc(bytes)) != 0 || (rc = d_out.alloc(bytes)) != 0) return rc;
    CU(cudaMemcpyAsync(d_in, in, bytes, cudaMemcpyHostToDevice, r->stream));
    if ((rc = launch_k5_full(r->d.p, r->tab.plan, r->tab.spec.k5, d_in, d_out, count, r->stream)) != 0) return rc;
    ++r->launches;
    CU(cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, r->stream));
    CU(cudaStreamSynchronize(r->stream));
    return 0;
}

int glava_b200_raster_textures(glava_b200* r, const uint16_t* tex_l, const uint16_t* tex_r) {
    clear_error();
    if (!r || !tex_l) return fail(GLAVA_B200_EINVAL, "glava_b200_raster_textures: null argument");
    UpdateInput in = { UpdateInput::TEXTURES, "glava_b200_raster_textures", tex_l, tex_r };
    int rc = check_update(r, in);
    if (rc) return rc;
    const size_t row = (size_t) r->d.p.n * 2;
    CU(cudaStreamSynchronize(r->spec_stream));
    char* dst = (char*) tex_half(r, r->tex_cur);
    CU(cudaMemcpy2DAsync(dst, 2 * row, tex_l, row, row, (size_t) r->batch, cudaMemcpyHostToDevice, r->stream));
    if (tex_r) CU(cudaMemcpy2DAsync(dst + row, 2 * row, tex_r, row, row, (size_t) r->batch, cudaMemcpyHostToDevice, r->stream));
    return enqueue_raster(r);
}

int glava_b200_transform_smooth(glava_b200* r, float* planes, int count) {
    clear_error();
    if (!r || !planes || count < 1) return fail(GLAVA_B200_EINVAL, "glava_b200_transform_smooth: bad arguments");
    if (!r->d.p.transform_smooth) return fail(GLAVA_B200_EINVAL, "glava_b200_transform_smooth: the renderer was not created with transform_smooth");
    if (!r->built) return unbuilt();
    CU(cudaSetDevice(r->device));
    const size_t bytes = (size_t) count * r->d.p.n * 4;
    DevBuf<float> d;
    int rc = d.alloc(bytes);
    if (rc) return rc;
    CU(cudaMemcpyAsync(d, planes, bytes, cudaMemcpyHostToDevice, r->stream));
    if ((rc = launch_transform_smooth(d, r->d.p.n, r->tab.ts_tab, r->tab.ts_asz, r->tab.ts_lim, count, r->stream)) != 0) return rc;
    ++r->launches;
    CU(cudaMemcpyAsync(planes, d, bytes, cudaMemcpyDeviceToHost, r->stream));
    CU(cudaStreamSynchronize(r->stream));
    return 0;
}

}  // extern "C"

// ---- lifetime of individual streams: reset, save, load (DESIGN.md §4.8) ---------------------------------------------------
static_assert(GLB_STATE_HEADER_BYTES == GLAVA_B200_STATE_HEADER_BYTES, "one header size");
static_assert(sizeof(StateHeader) + sizeof(glava_b200_params) <= GLB_STATE_HEADER_BYTES, "header holds the parameters");
static const size_t kStateStageBytes = (size_t) 16 << 20;   // blob segments per staging half (two halves)
enum { SS_SAVE = 0, SS_LOAD = 1, SS_RESET = 2 };

static StateLayout state_layout(const glava_b200_params& p, int n_in) {
    StateLayout L;
    L.n = p.n; L.n_in = n_in; L.F = p.avg_frames; L.esz = p.accel_fft ? 2 : 4;
    L.chans = p.module == GLAVA_B200_MOD_WAVE ? 1 : 2;
    return L;
}

// The parameters a blob records and is checked against: the effective ones, fb_slots zeroed (it sizes no stream's state)
static void state_params(const glava_b200* r, glava_b200_params* out) {
    memset(out, 0, sizeof(*out));
    memcpy(out, &r->d.p, sizeof(*out));
    out->fb_slots = 0;
}

static int state_unavailable(const char* who) {
    return fail(GLAVA_B200_EINVAL, "%s: not available with keyframe interpolation active (setinterpolate): the keyframe rotation "
                                   "is per renderer", who);
}

static int state_check_streams(const glava_b200* r, const int* streams, int count, const char* who) {
    if (count < 0 || (count > 0 && !streams)) return fail(GLAVA_B200_EINVAL, "%s: bad arguments", who);
    std::vector<char> seen((size_t) r->batch, 0);
    for (int i = 0; i < count; ++i) {
        const int s = streams[i];
        if (s < 0 || s >= r->batch) return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, s, r->batch);
        if (seen[(size_t) s]) return fail(GLAVA_B200_EINVAL, "%s: stream %d listed twice", who, s);
        seen[(size_t) s] = 1;
    }
    return 0;
}

namespace glb {
int state_check_blobs(const glava_b200* r, const void* const* blobs, int count, const char* who) {
    const StateLayout L = state_layout(r->d.p, r->d.n_in);
    glava_b200_params want;
    state_params(r, &want);
    for (int i = 0; i < count; ++i) {
        if (!blobs[i]) return fail(GLAVA_B200_EINVAL, "%s: blob %d is null", who, i);
        StateHeader h;
        memcpy(&h, blobs[i], sizeof(h));
        if (h.magic != GLB_STATE_MAGIC) return fail(GLAVA_B200_EINVAL, "%s: blob %d is not a stream state (bad magic)", who, i);
        if (h.version != GLB_STATE_VERSION)
            return fail(GLAVA_B200_EINVAL, "%s: blob %d has format version %u, this library reads %u", who, i, h.version, GLB_STATE_VERSION);
        if (h.header_bytes != GLB_STATE_HEADER_BYTES || h.params_bytes != sizeof(glava_b200_params) || h.blob_bytes != ss_blob_bytes(L))
            return fail(GLAVA_B200_EINVAL, "%s: blob %d has the wrong size (%llu bytes, this renderer's streams take %zu)", who, i,
                        (unsigned long long) h.blob_bytes, ss_blob_bytes(L));
        if (memcmp((const char*) blobs[i] + sizeof(StateHeader), &want, sizeof(want)) != 0)
            return fail(GLAVA_B200_EINVAL, "%s: blob %d was saved from a renderer with other parameters", who, i);
    }
    return 0;
}
}  // namespace glb

// device staging, allocated on first use: halves of up to kStateStageBytes of segments plus the chunk table
static int state_staging(glava_b200* r, const StateLayout& L) {
    if (r->ev_sst_free[1].get()) return 0;                   // created last: both halves are complete
    const size_t seg = ss_segment_bytes(L);
    size_t k = kStateStageBytes / seg;
    if (k < 1) k = 1;
    if (k > (size_t) r->batch) k = (size_t) r->batch;
    r->sst_streams = (int) k;
    r->sst_table = (k * 8 + 255) / 256 * 256;
    int rc;
    for (int i = 0; i < 2; ++i)
        if ((rc = r->d_sst[i].alloc(r->sst_table + k * seg)) != 0 || (rc = r->h_sst[i].alloc(k * 8)) != 0 ||
            (rc = r->ev_sst_copied[i].create()) != 0 || (rc = r->ev_sst_free[i].create()) != 0) return rc;
    return 0;
}

// Save / load / reset of the listed streams in chunks of at most sst_streams.  Kernels and D2H copies run on spec_stream
// (where every update reads and writes this state, in issue order); the H2D copies of load and reset run on copy_stream, so
// the host waits for copies only, never for earlier kernels.  Reset and load write the texture half the last raster may still
// read: spec_stream waits for that raster on the device.
static int state_io(glava_b200* r, int op, const int* streams, int count, void* const* out, const void* const* in) {
    const StateLayout L = state_layout(r->d.p, r->d.n_in);
    const size_t seg = ss_segment_bytes(L), blob = ss_blob_bytes(L);
    int rc;
    if (count == 0) return 0;
    if ((rc = state_staging(r, L)) != 0) return rc;
    StatePtrs P;
    P.gravity = (char*) (r->d.p.accel_fft ? (void*) r->d_gr_store : (void*) r->d_applied);
    P.ring = (char*) (r->d.p.accel_fft ? (void*) r->d_ring_u : (void*) r->d_ring_f);
    P.spec = (char*) r->d_spec.get(); P.tex = (char*) tex_half(r, r->tex_cur); P.av = (char*) r->d_av.get();
    P.fifo[0] = (char*) r->d_ring[r->ring_cur][0].get(); P.fifo[1] = (char*) r->d_ring[r->ring_cur][1].get();
    CU(cudaStreamWaitEvent(r->spec_stream, r->ev_raster_done[r->tex_cur], 0));
    const uint32_t F = (uint32_t) r->d.p.avg_frames;
    int last = -1;
    for (int c0 = 0; c0 < count; c0 += r->sst_streams) {
        const int k = r->sst_cur, cnt = count - c0 < r->sst_streams ? count - c0 : r->sst_streams;
        r->sst_cur ^= 1; last = k;
        CU(cudaEventSynchronize(r->ev_sst_copied[k]));          // the last table copy out of h_sst[k] (two chunks ago)
        int* tab = r->h_sst[k];
        for (int i = 0; i < cnt; ++i) {
            const int s = streams[c0 + i];
            tab[i] = s;
            tab[cnt + i] = (int) (r->desync ? r->cursor[(size_t) s] : (uint32_t) (r->updates % (unsigned long long) F));
        }
        char* d_tab = (char*) r->d_sst[k];
        char* d_seg = d_tab + r->sst_table;
        cudaStream_t up = op == SS_SAVE ? r->spec_stream : r->copy_stream;
        if (op != SS_SAVE) CU(cudaStreamWaitEvent(up, r->ev_sst_free[k], 0));
        CU(cudaMemcpyAsync(d_tab, tab, (size_t) cnt * 8, cudaMemcpyHostToDevice, up));
        if (op == SS_LOAD) {
            // runs of blobs adjacent in host memory go up as one strided copy each
            for (int i = 0; i < cnt;) {
                int j = i + 1;
                while (j < cnt && (const char*) in[c0 + j] == (const char*) in[c0 + j - 1] + blob) ++j;
                CU(cudaMemcpy2DAsync(d_seg + (size_t) i * seg, seg, (const char*) in[c0 + i] + GLB_STATE_HEADER_BYTES, blob, seg,
                                     (size_t) (j - i), cudaMemcpyHostToDevice, up));
                i = j;
            }
        }
        CU(cudaEventRecord(r->ev_sst_copied[k], up));
        if (op != SS_SAVE) CU(cudaStreamWaitEvent(r->spec_stream, r->ev_sst_copied[k], 0));
        if (op == SS_SAVE) rc = launch_state_pack(L, P, (const int*) d_tab, cnt, d_seg, r->spec_stream);
        else rc = launch_state_unpack(L, P, (const int*) d_tab, cnt, op == SS_LOAD ? d_seg : nullptr, r->spec_stream);
        if (rc) return rc;
        ++r->launches;
        if (op == SS_SAVE) {
            for (int i = 0; i < cnt;) {
                int j = i + 1;
                while (j < cnt && (char*) out[c0 + j] == (char*) out[c0 + j - 1] + blob) ++j;
                CU(cudaMemcpy2DAsync((char*) out[c0 + i] + GLB_STATE_HEADER_BYTES, blob, d_seg + (size_t) i * seg, seg, seg,
                                     (size_t) (j - i), cudaMemcpyDeviceToHost, r->spec_stream));
                i = j;
            }
        }
        CU(cudaEventRecord(r->ev_sst_free[k], r->spec_stream));
    }
    if (last < 0) return 0;
    if (op == SS_SAVE) {
        CU(cudaEventSynchronize(r->ev_sst_free[last]));
    } else {
        // a raster-only update after this call waits for ev_spec_done[tex_cur]: move it behind the new texture contents
        CU(cudaEventRecord(r->ev_spec_done[r->tex_cur], r->spec_stream));
        if (op == SS_LOAD) CU(cudaEventSynchronize(r->ev_sst_copied[last]));   // copy_stream runs in order: every blob is consumed
    }
    return 0;
}

namespace glb {
int state_save_ptrs(glava_b200* r, const int* streams, int count, void* const* blobs) {
    const char* who = "glava_b200_save_streams";
    if (r->d.interp_on) return state_unavailable(who);
    int rc = state_check_streams(r, streams, count, who);
    if (rc) return rc;
    for (int i = 0; i < count; ++i) if (!blobs[i]) return fail(GLAVA_B200_EINVAL, "%s: null blob", who);
    CU(cudaSetDevice(r->device));
    const StateLayout L = state_layout(r->d.p, r->d.n_in);
    StateHeader h;
    memset(&h, 0, sizeof(h));
    h.magic = GLB_STATE_MAGIC; h.version = GLB_STATE_VERSION; h.header_bytes = GLB_STATE_HEADER_BYTES;
    h.params_bytes = sizeof(glava_b200_params); h.blob_bytes = ss_blob_bytes(L);
    glava_b200_params q;
    state_params(r, &q);
    for (int i = 0; i < count; ++i) {
        char* b = (char*) blobs[i];
        memset(b, 0, GLB_STATE_HEADER_BYTES);
        memcpy(b, &h, sizeof(h));
        memcpy(b + sizeof(h), &q, sizeof(q));
    }
    return state_io(r, SS_SAVE, streams, count, blobs, nullptr);
}
int state_load_ptrs(glava_b200* r, const int* streams, int count, const void* const* blobs) {
    const char* who = "glava_b200_load_streams";
    if (r->d.interp_on) return state_unavailable(who);
    int rc = state_check_streams(r, streams, count, who);
    if (rc) return rc;
    if ((rc = state_check_blobs(r, blobs, count, who)) != 0) return rc;
    CU(cudaSetDevice(r->device));
    return state_io(r, SS_LOAD, streams, count, nullptr, blobs);
}
}  // namespace glb

extern "C" {

size_t glava_b200_stream_state_bytes(const glava_b200_params* p) {
    clear_error();
    if (!p) { fail(GLAVA_B200_EINVAL, "glava_b200_stream_state_bytes: null argument"); return 0; }
    if (validate_params(p) != 0) return 0;
    const Derived d = derive(*p);
    if (d.interp_on) { state_unavailable("glava_b200_stream_state_bytes"); return 0; }
    return ss_blob_bytes(state_layout(d.p, d.n_in));
}

int glava_b200_reset_streams(glava_b200* r, const uint8_t* mask) {
    clear_error();
    if (!r || !mask) return fail(GLAVA_B200_EINVAL, "glava_b200_reset_streams: null argument");
    if (r->d.interp_on) return state_unavailable("glava_b200_reset_streams");
    std::vector<int> list;
    for (int s = 0; s < r->batch; ++s) if (mask[s]) list.push_back(s);
    if (list.empty()) return 0;
    CU(cudaSetDevice(r->device));
    return state_io(r, SS_RESET, list.data(), (int) list.size(), nullptr, nullptr);
}

int glava_b200_save_streams(glava_b200* r, const int* streams, int count, void* blobs) {
    clear_error();
    if (!r || (count > 0 && !blobs)) return fail(GLAVA_B200_EINVAL, "glava_b200_save_streams: null argument");
    const size_t bytes = ss_blob_bytes(state_layout(r->d.p, r->d.n_in));
    std::vector<void*> ptrs(count > 0 ? (size_t) count : 0);
    for (size_t i = 0; i < ptrs.size(); ++i) ptrs[i] = (char*) blobs + i * bytes;
    return state_save_ptrs(r, streams, count, ptrs.data());
}

int glava_b200_load_streams(glava_b200* r, const int* streams, int count, const void* blobs) {
    clear_error();
    if (!r || (count > 0 && !blobs)) return fail(GLAVA_B200_EINVAL, "glava_b200_load_streams: null argument");
    const size_t bytes = ss_blob_bytes(state_layout(r->d.p, r->d.n_in));
    std::vector<const void*> ptrs(count > 0 ? (size_t) count : 0);
    for (size_t i = 0; i < ptrs.size(); ++i) ptrs[i] = (const char*) blobs + i * bytes;
    return state_load_ptrs(r, streams, count, ptrs.data());
}

}  // extern "C"

// ---- stream styles (DESIGN 4.9) ------------------------------------------------------------------------------------------
extern "C" {

int glava_b200_set_stream_styles(glava_b200* r, const int* streams, int count, const glava_b200_stream_style* styles) {
    clear_error();
    const char* who = "glava_b200_set_stream_styles";
    if (!r || (count > 0 && !styles)) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = state_check_streams(r, streams, count, who);
    if (rc) return rc;
    std::vector<glava_b200_stream_style> next = r->styles;
    if (next.empty()) next.assign((size_t) r->batch, style_key(glava_b200_stream_style{}, 0));
    for (int i = 0; i < count; ++i) next[(size_t) streams[i]] = styles[i];
    bool any = false;
    for (const glava_b200_stream_style& s : next) any |= s.set != 0;
    if (!any) next.clear();
    CU(cudaSetDevice(r->device));
    if ((rc = rebuild(r, r->d.user, next)) != 0) return rc;     // refuses an invalid style before it touches anything
    r->styles = std::move(next);
    return 0;
}

int glava_b200_get_stream_styles(const glava_b200* r, const int* streams, int count, glava_b200_stream_style* out) {
    clear_error();
    const char* who = "glava_b200_get_stream_styles";
    if (!r || (count > 0 && !out)) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    int rc = state_check_streams(r, streams, count, who);
    if (rc) return rc;
    for (int i = 0; i < count; ++i) {
        if (r->styles.empty()) memset(&out[i], 0, sizeof(out[i]));
        else out[i] = r->styles[(size_t) streams[i]];
    }
    return 0;
}

}  // extern "C"


// ---- what export.cpp reads of a renderer (DESIGN 4.10) -------------------------------------------------------------------
namespace glb {
RendererView renderer_view(glava_b200* r) {
    RendererView v;
    v.built = r->built; v.device = r->device; v.batch = r->batch; v.slots = r->slots;
    v.w = r->d.p.w; v.h = r->d.p.h; v.native = r->d.p.premultiply_alpha != 0; v.mark_key = r->mark_key;
    v.stream = r->stream; v.fb = r->frame.fb; v.marks = r->frame.marks;
    v.launches = &r->launches; v.attach = &r->attach; v.attach_free = &r->attach_free;
    return v;
}
}  // namespace glb
