// fakecuda.cpp — TEST INFRASTRUCTURE: the CUDA runtime calls of capi.cu and the kernel launchers it calls, on the host.
//
// tests/fakecuda/__init__.py compiles capi.cu and config.cpp with g++ against this file.  Host memory stands in for device
// and pinned memory; copies and kernels do nothing.  The runtime half counts the live buffers, pinned buffers, events and
// streams, fails the k-th resource creation on request, and records every error for cudaGetLastError as the runtime does
// (until read).  One device, 132 SMs, no PCI bus id.  The launcher half checks that every table the launch structure names
// exists, and reports a pending runtime error as its launch failure, as the real launchers' post-launch check does.
// Between fake_trace_begin and fake_trace_end both halves write a trace of the calls that enqueue work or wait for it
// (launches, copies, fills, event records and waits, synchronisations), one line each, with streams and events numbered
// in the order they were created since fake_trace_begin (s0: the legacy default stream).  launch_polar_geo records the
// parameters and the box of every call, so that a test can check which geometry caches the rebuild path asks for.
#include <cuda_runtime.h>

#include "../../glava_b200/csrc/internal.h"
#include "../../glava_b200/csrc/spectrum_plan.h"
#include "../../glava_b200/csrc/raster_plan.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace {
enum Kind { BUF, PINNED, EVENT, STREAM, KINDS };
std::set<void*> g_live[KINDS];
long g_creations = 0, g_fail_at = -1;
cudaError_t g_last = cudaSuccess;
long g_launches = 0, g_violations = 0, g_stale = 0, g_reached = 0;
std::string g_violation;
bool g_tracing = false;
std::string g_trace;
std::map<const void*, int> g_ids[KINDS];
int g_next_id[KINDS];
struct GeoCall { glava_b200_params p; int box[4]; int misalign; };
std::vector<GeoCall> g_geo;

void trace(const char* fmt, ...) {
    if (!g_tracing) return;
    char buf[256];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_trace += buf;
    g_trace += '\n';
}
std::string name(Kind k, const void* p) {
    if (!p && k == STREAM) return "s0";
    auto it = g_ids[k].find(p);
    return std::string(k == STREAM ? "s" : "e") + (it == g_ids[k].end() ? std::string("?") : std::to_string(it->second));
}
const char* kind_name(cudaMemcpyKind kind) {
    switch (kind) {
    case cudaMemcpyHostToDevice: return "H2D";
    case cudaMemcpyDeviceToHost: return "D2H";
    case cudaMemcpyDeviceToDevice: return "D2D";
    case cudaMemcpyHostToHost: return "H2H";
    default: return "default";
    }
}

cudaError_t record(cudaError_t e) {
    if (e != cudaSuccess) g_last = e;
    return e;
}
cudaError_t create(Kind k, void** out, size_t bytes) {
    *out = nullptr;
    if (g_creations++ == g_fail_at) return record(k == BUF || k == PINNED ? cudaErrorMemoryAllocation : cudaErrorLaunchOutOfResources);
    void* p = calloc(1, bytes ? bytes : 1);
    g_live[k].insert(p);
    g_ids[k][p] = ++g_next_id[k];
    *out = p;
    return cudaSuccess;
}
cudaError_t destroy(Kind k, void* p, bool null_ok) {
    if (!p && null_ok) return cudaSuccess;
    if (!g_live[k].erase(p)) return record(cudaErrorInvalidValue);
    g_ids[k].erase(p);
    free(p);
    return cudaSuccess;
}
cudaError_t handle(Kind k, const void* p) { return g_live[k].count(const_cast<void*>(p)) ? cudaSuccess : record(cudaErrorInvalidResourceHandle); }
cudaError_t stream_ok(cudaStream_t s) { return s ? handle(STREAM, s) : cudaSuccess; }

// which tables the launches have used, for the test to check that a configuration reaches what it is meant to
enum Reached { R_NEED = 1, R_TAPS = 2, R_FULL = 4, R_NEED_SMEM = 8, R_NEED_L2 = 16, R_GEO = 32, R_CTILE = 64, R_COLTAB = 128,
               R_TSMOOTH = 256 };

int launched(const char* what, void* stream, bool tables_ok, long reached = 0) {
    trace("launch %s %s", what, name(STREAM, stream).c_str());
    ++g_launches;
    g_reached |= reached;
    if (!tables_ok) {
        if (!g_violations) g_violation = what;
        ++g_violations;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        ++g_stale;
        return glb::fail(GLAVA_B200_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
    }
    return 0;
}
}  // namespace

// ---- the runtime -------------------------------------------------------------------------------------------------------
extern "C" {
const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : e == cudaErrorMemoryAllocation ? "out of memory" : "fake error"; }
cudaError_t cudaGetLastError(void) { const cudaError_t e = g_last; g_last = cudaSuccess; return e; }
cudaError_t cudaGetDeviceCount(int* count) { *count = 1; return cudaSuccess; }
cudaError_t cudaGetDevice(int* device) { *device = 0; return cudaSuccess; }
cudaError_t cudaSetDevice(int device) { return device == 0 ? cudaSuccess : record(cudaErrorInvalidDevice); }
cudaError_t cudaDeviceGetAttribute(int* value, enum cudaDeviceAttr attr, int) {
    *value = attr == cudaDevAttrMultiProcessorCount ? 132 : 0;
    return cudaSuccess;
}
cudaError_t cudaGetDeviceProperties(struct cudaDeviceProp* prop, int) { *prop = cudaDeviceProp(); prop->multiProcessorCount = 132; return cudaSuccess; }
cudaError_t cudaDeviceGetPCIBusId(char*, int, int) { return record(cudaErrorNotSupported); }
cudaError_t cudaDeviceGetStreamPriorityRange(int* least, int* greatest) { *least = 0; *greatest = -5; return cudaSuccess; }
cudaError_t cudaDeviceSetLimit(enum cudaLimit, size_t) { return cudaSuccess; }

cudaError_t cudaMalloc(void** p, size_t bytes) { return create(BUF, p, bytes); }
cudaError_t cudaFree(void* p) { return destroy(BUF, p, true); }
cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned int) { return create(PINNED, p, bytes); }
cudaError_t cudaFreeHost(void* p) { return destroy(PINNED, p, true); }
cudaError_t cudaHostRegister(void*, size_t, unsigned int) { return record(cudaErrorNotSupported); }
cudaError_t cudaHostUnregister(void*) { return record(cudaErrorNotSupported); }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned int) { return create(EVENT, (void**) e, 1); }
cudaError_t cudaEventCreate(cudaEvent_t* e) { return create(EVENT, (void**) e, 1); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { return destroy(EVENT, e, false); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned int) { return create(STREAM, (void**) s, 1); }
cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned int, int) { return create(STREAM, (void**) s, 1); }
cudaError_t cudaStreamDestroy(cudaStream_t s) { return destroy(STREAM, s, false); }

cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) {
    trace("record %s %s", name(EVENT, e).c_str(), name(STREAM, s).c_str());
    cudaError_t r = handle(EVENT, e); return r ? r : stream_ok(s); }
cudaError_t cudaEventSynchronize(cudaEvent_t e) {
    trace("event_sync %s", name(EVENT, e).c_str());
    return handle(EVENT, e); }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = 0.0f;
    cudaError_t r = handle(EVENT, a);
    return r ? r : handle(EVENT, b);
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned int) {
    trace("wait %s %s", name(STREAM, s).c_str(), name(EVENT, e).c_str());
    cudaError_t r = handle(EVENT, e); return r ? r : stream_ok(s); }
cudaError_t cudaStreamSynchronize(cudaStream_t s) {
    trace("stream_sync %s", name(STREAM, s).c_str());
    return stream_ok(s); }
cudaError_t cudaStreamSetAttribute(cudaStream_t s, cudaStreamAttrID, const cudaStreamAttrValue*) { return stream_ok(s); }
cudaError_t cudaMemsetAsync(void* p, int, size_t bytes, cudaStream_t s) {
    trace("memset %zu %s", bytes, name(STREAM, s).c_str());
    return p ? stream_ok(s) : record(cudaErrorInvalidValue);
}
cudaError_t cudaMemcpyAsync(void* d, const void* src, size_t bytes, enum cudaMemcpyKind kind, cudaStream_t s) {
    trace("memcpy %s %zu %s", kind_name(kind), bytes, name(STREAM, s).c_str());
    return d && src ? stream_ok(s) : record(cudaErrorInvalidValue);
}
cudaError_t cudaMemcpy2DAsync(void* d, size_t, const void* src, size_t, size_t width, size_t height, enum cudaMemcpyKind kind,
                              cudaStream_t s) {
    trace("memcpy2d %s %zux%zu %s", kind_name(kind), width, height, name(STREAM, s).c_str());
    return d && src ? stream_ok(s) : record(cudaErrorInvalidValue);
}
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { *h = cudaIpcMemHandle_t(); return handle(BUF, p); }

// ---- the test's controls -----------------------------------------------------------------------------------------------
// fail the k-th resource creation from now on (k < 0: none); counting restarts
void fake_fail_at(long k) { g_fail_at = k; g_creations = 0; }
long fake_creations(void) { return g_creations; }
long fake_live(int kind) { return (long) g_live[kind].size(); }
long fake_launches(void) { return g_launches; }
long fake_violations(void) { return g_violations; }
const char* fake_first_violation(void) { return g_violation.c_str(); }
long fake_stale(void) { return g_stale; }
long fake_reached(void) { return g_reached; }
void fake_clear(void) { g_launches = g_violations = g_stale = g_reached = 0; g_violation.clear(); g_last = cudaSuccess; g_geo.clear(); }
// the launch_polar_geo calls since fake_clear: their count, and call i's parameters and box; returns the cache address
// modulo 16, which must be 0 for its int4 entries (the fake's buffers are 16-byte aligned, as cudaMalloc's are), or -1: no
// such call
long fake_geo_calls(void) { return (long) g_geo.size(); }
int fake_geo_call(long i, glava_b200_params* p, int* box) {
    if (i < 0 || i >= (long) g_geo.size()) return -1;
    *p = g_geo[(size_t) i].p;
    for (int k = 0; k < 4; ++k) box[k] = g_geo[(size_t) i].box[k];
    return g_geo[(size_t) i].misalign;
}
// start a trace: streams and events are numbered from 1 in the order they are created from now on
void fake_trace_begin(void) {
    g_trace.clear();
    for (int k = 0; k < KINDS; ++k) { g_ids[k].clear(); g_next_id[k] = 0; }
    g_tracing = true;
}
void fake_trace_end(void) { g_tracing = false; }
const char* fake_trace(void) { return g_trace.c_str(); }
}  // extern "C"

// ---- the launchers capi.cu calls ---------------------------------------------------------------------------------------
namespace glb {
int launch_spectrum_update(const glava_b200_params&, const SpectrumPlan& pl, const SpectrumDevTables& t, const SpectrumArgs& a, void* st) {
    const bool ok = (!pl.need_list || t.need) && (!pl.tap_table || (t.tap_tab && t.csr)) &&
                    (pl.k5 != K5Form::NEED_SMEM || t.need_blk) && (pl.k5 != K5Form::NEED_L2 || t.av_t) &&
                    (!pl.full_table || t.k5.blk) && a.spec && a.tex;
    const long reached = (pl.need_list ? R_NEED : 0) | (pl.tap_table ? R_TAPS : 0) | (pl.full_table ? R_FULL : 0) |
                         (pl.k5 == K5Form::NEED_SMEM ? R_NEED_SMEM : 0) | (pl.k5 == K5Form::NEED_L2 ? R_NEED_L2 : 0);
    const int rc = launched("spectrum update", st, ok, reached);
    return rc ? rc : 1;
}
int launch_k5_full(const glava_b200_params&, const SpectrumPlan& pl, const K5Table& t, const uint16_t* in, uint16_t* out, int, void* st) {
    return launched("whole-plane K5", st, (!pl.full_table || t.blk) && in && out);
}
int launch_raster(const glava_b200_params&, const RasterPlan& pl, const RasterArgs& a, void* st) {
    const bool ok = (!pl.geo || a.geo) && (!pl.ctile || (a.ctile && a.ctile_zero)) && (!pl.coltab || a.coltab) &&
                    (!pl.rowtab || a.rowtab) && a.fb && a.marks && a.tex;
    return launched("raster", st, ok, (pl.geo ? R_GEO : 0) | (pl.ctile ? R_CTILE : 0) | (pl.coltab ? R_COLTAB : 0));
}
int launch_bars_rowtab(const glava_b200_params&, void* d_rowtab, void* st) { return launched("row table", st, d_rowtab != nullptr); }
int launch_texmm(const glava_b200_params&, const uint16_t* tex, uint32_t* out, int, void* st) { return launched("texmm", st, tex && out); }
int launch_polar_geo(const glava_b200_params& p, void* d_geo, const int* box, void* st) {
    GeoCall c;
    c.p = p;
    for (int k = 0; k < 4; ++k) c.box[k] = box[k];
    c.misalign = (int) ((uintptr_t) d_geo % 16);
    g_geo.push_back(c);
    return launched("polar geometry", st, d_geo != nullptr);
}
size_t circle_tile_bytes(const glava_b200_params& p, int* ntx, int* nty) {
    *ntx = (p.w + 127) / 128; *nty = (p.h + 7) / 8;
    return (size_t) *ntx * *nty * (sizeof(int4) + sizeof(int));
}
int launch_circle_tiles(const glava_b200_params&, const void* d_geo, const int*, void* d_tiles, void* st) {
    return launched("circle tiles", st, d_geo && d_tiles);
}
int launch_fifo_ingest(const glava_b200_params&, const void* chunks, bool, int, const float* sl, const float* sr, float* dl, float* dr, int,
                       void* st) {
    return launched("fifo ingest", st, chunks && sl && sr && dl && dr);
}
int launch_bufscale(const float* il, const float*, float* ol, float* orr, int, int, int, int, void* st) {
    return launched("bufscale", st, il && ol && orr);
}
int launch_transform_smooth(float* planes, int, const void* tab, int, int, int, void* st, const uint32_t*, int) {
    return launched("transform_smooth", st, planes && tab, R_TSMOOTH);
}
int launch_upload(const float* s, const float*, float, uint16_t* out, size_t, void* st) { return launched("upload", st, s && out); }
int launch_state_pack(const StateLayout&, const StatePtrs&, const int* table, int, void* out, void* st) {
    return launched("state pack", st, table && out);
}
int launch_state_unpack(const StateLayout&, const StatePtrs&, const int* table, int, const void*, void* st) {
    return launched("state unpack", st, table != nullptr);
}
}  // namespace glb
