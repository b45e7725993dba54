// sharded.cpp — one handle for a batch spread over several GPUs of a node (SURVEY §8b's `device_mask`).
//
// The streams of a batch are independent (every GLava process renders its own), so the batch is cut into contiguous
// blocks, one per device, and nothing ever crosses between devices: no collective, no peer copies.  What this file adds
// over N single-device handles is the plumbing a GLava-side caller would otherwise write: one worker thread per device
// (pinned to the device's NUMA node, so its pinned staging and its launches are local), a broadcast of every call to all
// shards at once (the per-device H2D copies and launches are issued concurrently, not one device after another), and
// stream-indexed read-backs.  Host code only: every device operation goes through the single-device C ABI (capi.cu).
#include "internal.h"

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <string>
#include <mutex>
#include <thread>
#include <vector>

using namespace glb;

namespace {

struct Shard {
    glava_b200* r = nullptr;
    int device = 0, first = 0, count = 0;
    std::thread th;
    std::mutex mu; std::condition_variable cv;
    std::function<int(Shard&)> job; bool has_job = false, quit = false, done = true;
    int rc = 0;
    std::string err;
};

}  // namespace

struct glava_b200_sharded {
    int batch = 0;
    glava_b200_params p;
    std::vector<Shard*> shards;
};

// contiguous block partition, counts differ by at most one (the arithmetic of glava_b200/shard.py shard_streams)
extern "C" int glava_b200_shard_range(int batch, int shards, int k, int* first, int* count) {
    if (batch < 0 || shards < 1 || k < 0 || k >= shards || !first || !count) return fail(GLAVA_B200_EINVAL, "glava_b200_shard_range: bad arguments");
    const int base = batch / shards, extra = batch % shards;
    *count = base + (k < extra ? 1 : 0);
    *first = k * base + (k < extra ? k : extra);
    return 0;
}

static void worker(Shard* s) {
    glava_b200_bind_thread_to_device(s->device);            // launches and pinned staging from the device's own socket
    for (;;) {
        std::function<int(Shard&)> job;
        {
            std::unique_lock<std::mutex> lk(s->mu);
            s->cv.wait(lk, [&] { return s->has_job || s->quit; });
            if (s->quit && !s->has_job) return;
            job = s->job; s->has_job = false;
        }
        clear_error();
        const int rc = job(*s);
        {
            std::lock_guard<std::mutex> lk(s->mu);
            s->rc = rc;
            s->err = rc ? glava_b200_last_error() : "";
            s->done = true;
        }
        s->cv.notify_all();
    }
}

// run `fn` on every shard's worker at once; returns the first failure (its message becomes this thread's last error)
static int broadcast(glava_b200_sharded* g, const std::function<int(Shard&)>& fn) {
    for (Shard* s : g->shards) {
        std::lock_guard<std::mutex> lk(s->mu);
        s->job = fn; s->has_job = true; s->done = false;
        s->cv.notify_all();
    }
    int rc = 0;
    for (Shard* s : g->shards) {
        std::unique_lock<std::mutex> lk(s->mu);
        s->cv.wait(lk, [&] { return s->done; });
        if (s->rc && !rc) rc = fail(s->rc, "device %d (streams %d..%d): %s", s->device, s->first, s->first + s->count - 1, s->err.c_str());
    }
    return rc;
}

extern "C" {

void glava_b200_sharded_destroy(glava_b200_sharded* g) {
    if (!g) return;
    for (Shard* s : g->shards) {
        if (s->th.joinable()) {
            { std::lock_guard<std::mutex> lk(s->mu); s->job = [](Shard& q) { if (q.r) glava_b200_destroy(q.r); q.r = nullptr; return 0; }; s->has_job = true; s->done = false; s->quit = true; }
            s->cv.notify_all();
            s->th.join();
        }
        if (s->r) glava_b200_destroy(s->r);
        delete s;
    }
    delete g;
}

// `devices`: n CUDA device ordinals, one shard each (an ordinal may repeat: several shards on one device).
glava_b200_sharded* glava_b200_new_sharded_devices(const glava_b200_params* params, int batch, const int* devices, int n) {
    clear_error();
    if (!params || !devices || n < 1 || batch < n) { fail(GLAVA_B200_EINVAL, "glava_b200_new_sharded: need 1 <= devices <= batch"); return nullptr; }
    glava_b200_sharded* g = new glava_b200_sharded();
    g->batch = batch; g->p = *params;
    for (int k = 0; k < n; ++k) {
        Shard* s = new Shard();
        s->device = devices[k];
        glava_b200_shard_range(batch, n, k, &s->first, &s->count);
        g->shards.push_back(s);
        s->th = std::thread(worker, s);
    }
    const glava_b200_params pp = *params;
    const int rc = broadcast(g, [pp](Shard& s) {
        s.r = glava_b200_new(&pp, s.count, s.device);
        return s.r ? 0 : GLAVA_B200_ECUDA;
    });
    if (rc) { glava_b200_sharded_destroy(g); return nullptr; }
    return g;
}

// device_mask: bit d set = CUDA device d takes a shard (ascending order); 0 = every visible device.
glava_b200_sharded* glava_b200_new_sharded(const glava_b200_params* params, int batch, uint64_t device_mask) {
    clear_error();
    std::vector<int> devs;
    if (device_mask == 0) {
        const int n = glava_b200_device_count();
        for (int d = 0; d < n; ++d) devs.push_back(d);
    } else {
        for (int d = 0; d < 64; ++d) if (device_mask & (1ull << d)) devs.push_back(d);
    }
    if (devs.empty()) { fail(GLAVA_B200_ECUDA, "no CUDA device available: the GPU path has no CPU fallback"); return nullptr; }
    while ((int) devs.size() > batch) devs.pop_back();
    return glava_b200_new_sharded_devices(params, batch, devs.data(), (int) devs.size());
}

int glava_b200_sharded_shards(const glava_b200_sharded* g) { return g ? (int) g->shards.size() : 0; }
int glava_b200_sharded_batch(const glava_b200_sharded* g) { return g ? g->batch : 0; }
glava_b200* glava_b200_sharded_shard(const glava_b200_sharded* g, int k, int* device, int* first_stream, int* count) {
    if (!g || k < 0 || k >= (int) g->shards.size()) return nullptr;
    const Shard* s = g->shards[k];
    if (device) *device = s->device;
    if (first_stream) *first_stream = s->first;
    if (count) *count = s->count;
    return s->r;
}

// rd_update for the whole batch: lb / rb HOST [batch][bsz]; modified: NULL = every stream, else one byte per stream.
int glava_b200_sharded_update(glava_b200_sharded* g, const float* lb, const float* rb, size_t bsz, const uint8_t* modified) {
    clear_error();
    if (!g || !lb) return fail(GLAVA_B200_EINVAL, "glava_b200_sharded_update: null argument");
    return broadcast(g, [=](Shard& s) {
        const float* l = lb + (size_t) s.first * bsz;
        const float* r = rb ? rb + (size_t) s.first * bsz : nullptr;
        return modified ? glava_b200_update_masked(s.r, l, r, bsz, modified + s.first) : glava_b200_update(s.r, l, r, bsz, 1);
    });
}
int glava_b200_sharded_rerender(glava_b200_sharded* g) {                    // rd_update(modified = false) for every stream
    clear_error();
    if (!g) return fail(GLAVA_B200_EINVAL, "null argument");
    return broadcast(g, [](Shard& s) { return glava_b200_update_rings(s.r, 0); });
}
// fifo.c:89-110 for the whole batch: chunks HOST [batch][frames * 2] int16, then the update on the resident rings
int glava_b200_sharded_ingest_fifo(glava_b200_sharded* g, const int16_t* chunks, int frames) {
    clear_error();
    if (!g || !chunks || frames < 1) return fail(GLAVA_B200_EINVAL, "glava_b200_sharded_ingest_fifo: bad arguments");
    return broadcast(g, [=](Shard& s) {
        const int rc = glava_b200_ingest_fifo(s.r, chunks + (size_t) s.first * frames * 2, frames);
        return rc ? rc : glava_b200_update_rings(s.r, 1);
    });
}
int glava_b200_sharded_sync(glava_b200_sharded* g) {
    clear_error();
    if (!g) return fail(GLAVA_B200_EINVAL, "null argument");
    return broadcast(g, [](Shard& s) { return glava_b200_sync(s.r); });
}
static Shard* shard_of(glava_b200_sharded* g, int stream) {
    if (!g || stream < 0 || stream >= g->batch) return nullptr;
    for (Shard* s : g->shards) if (stream >= s->first && stream < s->first + s->count) return s;
    return nullptr;
}
int glava_b200_sharded_readback(glava_b200_sharded* g, int stream, uint8_t* rgba) {
    clear_error();
    Shard* s = shard_of(g, stream);
    if (!s || !rgba) return fail(GLAVA_B200_EINVAL, "glava_b200_sharded_readback: bad arguments");
    return glava_b200_readback(s->r, stream - s->first, rgba);
}
// DEVICE pointer of a stream's latest frame and the device it lives on (for a consumer that stays in HBM)
const void* glava_b200_sharded_frame_device(glava_b200_sharded* g, int stream, int* device) {
    Shard* s = shard_of(g, stream);
    if (!s) return nullptr;
    if (device) *device = s->device;
    return glava_b200_frame_device(s->r, stream - s->first);
}
// Per-stream state (DESIGN.md §4.8), global stream indices: reset by each shard's slice of the mask; save and load group the
// listed streams per shard and run every shard's part at once.  Indices and blobs are checked for the whole call before any
// shard starts, so a rejected call touches no shard.
int glava_b200_sharded_reset_streams(glava_b200_sharded* g, const uint8_t* mask) {
    clear_error();
    if (!g || !mask) return fail(GLAVA_B200_EINVAL, "glava_b200_sharded_reset_streams: null argument");
    if (glava_b200_stream_state_bytes(&g->p) == 0) return GLAVA_B200_EINVAL;
    return broadcast(g, [=](Shard& s) { return glava_b200_reset_streams(s.r, mask + s.first); });
}

// split `streams` into per-shard local index lists and blob pointers (blob i at base + i * bytes)
static int group_streams(glava_b200_sharded* g, const int* streams, int count, const char* base, size_t bytes, const char* who,
                         std::vector<std::vector<int>>* idx, std::vector<std::vector<const char*>>* ptr) {
    if (count < 0 || (count > 0 && (!streams || !base))) return fail(GLAVA_B200_EINVAL, "%s: bad arguments", who);
    idx->assign(g->shards.size(), {}); ptr->assign(g->shards.size(), {});
    std::vector<char> seen((size_t) g->batch, 0);
    for (int i = 0; i < count; ++i) {
        const int s = streams[i];
        if (s < 0 || s >= g->batch) return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, s, g->batch);
        if (seen[(size_t) s]) return fail(GLAVA_B200_EINVAL, "%s: stream %d listed twice", who, s);
        seen[(size_t) s] = 1;
        for (size_t k = 0; k < g->shards.size(); ++k) {
            const Shard* sh = g->shards[k];
            if (s >= sh->first && s < sh->first + sh->count) {
                (*idx)[k].push_back(s - sh->first); (*ptr)[k].push_back(base + (size_t) i * bytes);
                break;
            }
        }
    }
    return 0;
}

int glava_b200_sharded_save_streams(glava_b200_sharded* g, const int* streams, int count, void* blobs) {
    clear_error();
    const char* who = "glava_b200_sharded_save_streams";
    if (!g) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    const size_t bytes = glava_b200_stream_state_bytes(&g->p);
    if (!bytes) return GLAVA_B200_EINVAL;
    std::vector<std::vector<int>> idx; std::vector<std::vector<const char*>> ptr;
    int rc = group_streams(g, streams, count, (const char*) blobs, bytes, who, &idx, &ptr);
    if (rc) return rc;
    return broadcast(g, [&](Shard& s) {
        const size_t k = (size_t) (std::find(g->shards.begin(), g->shards.end(), &s) - g->shards.begin());
        if (idx[k].empty()) return 0;
        std::vector<void*> out(ptr[k].size());
        for (size_t i = 0; i < out.size(); ++i) out[i] = (void*) ptr[k][i];
        return state_save_ptrs(s.r, idx[k].data(), (int) idx[k].size(), out.data());
    });
}

int glava_b200_sharded_load_streams(glava_b200_sharded* g, const int* streams, int count, const void* blobs) {
    clear_error();
    const char* who = "glava_b200_sharded_load_streams";
    if (!g) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    const size_t bytes = glava_b200_stream_state_bytes(&g->p);
    if (!bytes) return GLAVA_B200_EINVAL;
    std::vector<std::vector<int>> idx; std::vector<std::vector<const char*>> ptr;
    int rc = group_streams(g, streams, count, (const char*) blobs, bytes, who, &idx, &ptr);
    if (rc) return rc;
    for (size_t k = 0; k < g->shards.size(); ++k) {
        if (ptr[k].empty()) continue;
        std::vector<const void*> in(ptr[k].begin(), ptr[k].end());
        if ((rc = state_check_blobs(g->shards[k]->r, in.data(), (int) in.size(), who)) != 0) return rc;
    }
    return broadcast(g, [&](Shard& s) {
        const size_t k = (size_t) (std::find(g->shards.begin(), g->shards.end(), &s) - g->shards.begin());
        if (idx[k].empty()) return 0;
        std::vector<const void*> in(ptr[k].begin(), ptr[k].end());
        return state_load_ptrs(s.r, idx[k].data(), (int) idx[k].size(), in.data());
    });
}

// Per-stream styles (DESIGN 4.9), global stream indices.  Indices and styles are checked for the whole call before any
// shard starts, so a rejected call touches no shard.
int glava_b200_sharded_set_stream_styles(glava_b200_sharded* g, const int* streams, int count, const glava_b200_stream_style* styles) {
    clear_error();
    const char* who = "glava_b200_sharded_set_stream_styles";
    if (!g || (count > 0 && !styles)) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    std::vector<std::vector<int>> idx; std::vector<std::vector<const char*>> ptr;
    int rc = group_streams(g, streams, count, (const char*) styles, sizeof(glava_b200_stream_style), who, &idx, &ptr);
    if (rc) return rc;
    for (int i = 0; i < count; ++i) {
        glava_b200_params q;
        if ((rc = glava_b200_style_params(&g->p, &styles[i], &q)) != 0) return rc;
    }
    return broadcast(g, [&](Shard& s) {
        const size_t k = (size_t) (std::find(g->shards.begin(), g->shards.end(), &s) - g->shards.begin());
        if (idx[k].empty()) return 0;
        std::vector<glava_b200_stream_style> st(ptr[k].size());
        for (size_t i = 0; i < st.size(); ++i) st[i] = *(const glava_b200_stream_style*) ptr[k][i];
        return glava_b200_set_stream_styles(s.r, idx[k].data(), (int) idx[k].size(), st.data());
    });
}

int glava_b200_sharded_get_stream_styles(const glava_b200_sharded* g, const int* streams, int count, glava_b200_stream_style* out) {
    clear_error();
    const char* who = "glava_b200_sharded_get_stream_styles";
    if (!g || (count > 0 && !out)) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    glava_b200_sharded* gg = const_cast<glava_b200_sharded*>(g);
    std::vector<std::vector<int>> idx; std::vector<std::vector<const char*>> ptr;
    int rc = group_streams(gg, streams, count, (const char*) out, sizeof(glava_b200_stream_style), who, &idx, &ptr);
    if (rc) return rc;
    for (size_t k = 0; k < g->shards.size(); ++k) {
        if (idx[k].empty()) continue;
        std::vector<glava_b200_stream_style> st(idx[k].size());
        if ((rc = glava_b200_get_stream_styles(g->shards[k]->r, idx[k].data(), (int) idx[k].size(), st.data())) != 0) return rc;
        for (size_t i = 0; i < st.size(); ++i) *(glava_b200_stream_style*) ptr[k][i] = st[i];
    }
    return 0;
}

// The caller-buffer exports (DESIGN 4.10–4.12), global stream indices (repeats allowed): the list is split by shard, dst[i]
// and dst_uv[i] travelling with streams[i].  Every shard's part passes the single-renderer checks, and for an overlay the
// whole list the overlap test against itself and every shard's framebuffer (shards may share a device), before any shard
// starts; the shards then issue at once.  A ladder (rungs non-null) carries nrungs destinations per entry; an overlay's
// opacity (DESIGN 4.20, null: all 255) travels with its entry.
static int sharded_export(glava_b200_sharded* g, ExportKind kind, const int* streams, int count, void* const* dst,
                          void* const* dst_uv, const glava_b200_export* desc, const glava_b200_export_scale* scale, const char* who,
                          const glava_b200_export_rung* rungs = nullptr, int nrungs = 1, const uint8_t* opacity = nullptr) {
    clear_error();
    const bool ladder = kind == ExportKind::ladder;
    if (!g || (!ladder && !desc)) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    if (ladder) { const int rc = ladder_shape_check(rungs, nrungs, who); if (rc) return rc; }
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !dst) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    const size_t per = ladder ? (size_t) nrungs : 1;
    std::vector<std::vector<int>> idx(g->shards.size());
    std::vector<std::vector<void*>> ptr(g->shards.size()), uv(g->shards.size());
    std::vector<std::vector<uint8_t>> op(g->shards.size());
    for (int i = 0; i < count; ++i) {
        const int s = streams[i];
        if (s < 0 || s >= g->batch) return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, s, g->batch);
        for (size_t k = 0; k < g->shards.size(); ++k) {
            const Shard* sh = g->shards[k];
            if (s >= sh->first && s < sh->first + sh->count) {
                idx[k].push_back(s - sh->first);
                if (opacity) op[k].push_back(opacity[i]);
                for (size_t j = 0; j < per; ++j) {
                    ptr[k].push_back(dst[i * per + j]); uv[k].push_back(dst_uv ? dst_uv[i * per + j] : nullptr);
                }
                break;
            }
        }
    }
    std::vector<const uint8_t*> fb;
    std::vector<size_t> fb_bytes;
    for (size_t k = 0; k < g->shards.size(); ++k) {
        const RendererView v = renderer_view(g->shards[k]->r);
        fb.push_back(v.fb); fb_bytes.push_back((size_t) v.slots * (size_t) v.h * (size_t) v.w * 4);
        if (idx[k].empty()) continue;
        const int rc = ladder ? ladder_check(g->shards[k]->r, idx[k].data(), (int) idx[k].size(), rungs, nrungs, ptr[k].data(),
                                             dst_uv ? uv[k].data() : nullptr, who)
                              : export_check(kind, g->shards[k]->r, idx[k].data(), (int) idx[k].size(), ptr[k].data(),
                                             dst_uv ? uv[k].data() : nullptr, desc, scale, who);
        if (rc) return rc;
    }
    if (kind == ExportKind::overlay) {
        const RendererView v0 = renderer_view(g->shards[0]->r);
        const int rc = overlay_geometry_check(v0.w, v0.h, count, dst, dst_uv, *desc, fb.data(), fb_bytes.data(), (int) fb.size(), who);
        if (rc) return rc;
    }
    return broadcast(g, [&](Shard& s) {
        const size_t k = (size_t) (std::find(g->shards.begin(), g->shards.end(), &s) - g->shards.begin());
        if (idx[k].empty()) return 0;
        if (ladder)
            return ladder_run(s.r, idx[k].data(), (int) idx[k].size(), rungs, nrungs, ptr[k].data(), dst_uv ? uv[k].data() : nullptr,
                              nullptr, nullptr, who);
        return export_run(kind, s.r, idx[k].data(), (int) idx[k].size(), ptr[k].data(), dst_uv ? uv[k].data() : nullptr, desc,
                          scale, nullptr, nullptr, opacity ? op[k].data() : nullptr, opacity ? who : nullptr);
    });
}

int glava_b200_sharded_export_frames(glava_b200_sharded* g, const int* streams, int count, void* const* dst, const glava_b200_export* desc) {
    return sharded_export(g, ExportKind::frames, streams, count, dst, nullptr, desc, nullptr, "glava_b200_sharded_export_frames");
}
int glava_b200_sharded_export_scaled(glava_b200_sharded* g, const int* streams, int count, void* const* dst, void* const* dst_uv,
                                     const glava_b200_export* desc, const glava_b200_export_scale* scale) {
    return sharded_export(g, ExportKind::scaled, streams, count, dst, dst_uv, desc, scale, "glava_b200_sharded_export_scaled");
}
int glava_b200_sharded_overlay_frames(glava_b200_sharded* g, const int* streams, int count, void* const* dst, void* const* dst_uv,
                                      const glava_b200_export* desc) {
    return sharded_export(g, ExportKind::overlay, streams, count, dst, dst_uv, desc, nullptr, "glava_b200_sharded_overlay_frames");
}
int glava_b200_sharded_overlay_frames_opacity(glava_b200_sharded* g, const int* streams, int count, void* const* dst,
                                              void* const* dst_uv, const glava_b200_export* desc, const uint8_t* opacity) {
    return sharded_export(g, ExportKind::overlay, streams, count, dst, dst_uv, desc, nullptr, "glava_b200_sharded_overlay_frames_opacity",
                          nullptr, 1, opacity);
}
int glava_b200_sharded_export_ladder(glava_b200_sharded* g, const int* streams, int count, const glava_b200_export_rung* rungs,
                                     int nrungs, void* const* dst, void* const* dst_uv) {
    return sharded_export(g, ExportKind::ladder, streams, count, dst, dst_uv, nullptr, nullptr, "glava_b200_sharded_export_ladder",
                          rungs, nrungs);
}

// glava_b200_overlay_planes with global stream indices: the list split by shard (pics[i] and opacity[i] travelling with
// streams[i]), every shard's part checked as one renderer, then the whole list's overlap and every shard's framebuffer, before
// any shard starts.  scale non-null: glava_b200_overlay_scaled's (DESIGN 4.21), the rectangles out_w x out_h.
static int sharded_planes(glava_b200_sharded* g, const int* streams, int count, const glava_b200_picture* pics,
                          const glava_b200_overlay_planes_desc* desc, const uint8_t* opacity, const char* who,
                          const glava_b200_export_scale* scale = nullptr) {
    clear_error();
    if (!g || !desc) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    if (count < 1) return fail(GLAVA_B200_EINVAL, "%s: count %d < 1", who, count);
    if (!streams || !pics) return fail(GLAVA_B200_EINVAL, "%s: null argument", who);
    std::vector<std::vector<int>> idx(g->shards.size());
    std::vector<std::vector<glava_b200_picture>> part(g->shards.size());
    std::vector<std::vector<uint8_t>> op(g->shards.size());
    for (int i = 0; i < count; ++i) {
        const int s = streams[i];
        if (s < 0 || s >= g->batch) return fail(GLAVA_B200_EINVAL, "%s: stream %d out of range (batch %d)", who, s, g->batch);
        for (size_t k = 0; k < g->shards.size(); ++k) {
            const Shard* sh = g->shards[k];
            if (s >= sh->first && s < sh->first + sh->count) {
                idx[k].push_back(s - sh->first);
                part[k].push_back(pics[i]);
                if (opacity) op[k].push_back(opacity[i]);
                break;
            }
        }
    }
    std::vector<const uint8_t*> fb;
    std::vector<size_t> fb_bytes;
    const RendererView v0 = renderer_view(g->shards[0]->r);
    glava_b200_export_scale q = { 0, 0, v0.w, v0.h, v0.w, v0.h };   // every shard has the same frame size
    for (size_t k = 0; k < g->shards.size(); ++k) {
        const RendererView v = renderer_view(g->shards[k]->r);
        fb.push_back(v.fb); fb_bytes.push_back((size_t) v.slots * (size_t) v.h * (size_t) v.w * 4);
        if (idx[k].empty()) continue;
        const int rc = scale ? scaled_overlay_check(g->shards[k]->r, idx[k].data(), (int) idx[k].size(), part[k].data(), desc, scale,
                                                    &q, who)
                             : planes_check(g->shards[k]->r, idx[k].data(), (int) idx[k].size(), part[k].data(), desc, who);
        if (rc) return rc;
    }
    const int rc = planes_geometry_check(q.out_w, q.out_h, count, pics, *desc, fb.data(), fb_bytes.data(), (int) fb.size(), who,
                                         scale != nullptr);
    if (rc) return rc;
    return broadcast(g, [&](Shard& s) {
        const size_t k = (size_t) (std::find(g->shards.begin(), g->shards.end(), &s) - g->shards.begin());
        if (idx[k].empty()) return 0;
        if (scale)
            return scaled_overlay_run(s.r, idx[k].data(), (int) idx[k].size(), part[k].data(), desc, scale,
                                      opacity ? op[k].data() : nullptr, nullptr, nullptr, who);
        return planes_run(s.r, idx[k].data(), (int) idx[k].size(), part[k].data(), desc, nullptr, nullptr, who,
                          opacity ? op[k].data() : nullptr);
    });
}
int glava_b200_sharded_overlay_planes(glava_b200_sharded* g, const int* streams, int count, const glava_b200_picture* pics,
                                      const glava_b200_overlay_planes_desc* desc) {
    return sharded_planes(g, streams, count, pics, desc, nullptr, "glava_b200_sharded_overlay_planes");
}
int glava_b200_sharded_overlay_planes_opacity(glava_b200_sharded* g, const int* streams, int count, const glava_b200_picture* pics,
                                              const glava_b200_overlay_planes_desc* desc, const uint8_t* opacity) {
    return sharded_planes(g, streams, count, pics, desc, opacity, "glava_b200_sharded_overlay_planes_opacity");
}
int glava_b200_sharded_overlay_scaled(glava_b200_sharded* g, const int* streams, int count, const glava_b200_picture* pics,
                                      const glava_b200_overlay_planes_desc* desc, const glava_b200_export_scale* scale,
                                      const uint8_t* opacity) {
    if (!scale) {                                           // refused here: sharded_planes reads null as overlay_planes
        clear_error();
        return fail(GLAVA_B200_EINVAL, "glava_b200_sharded_overlay_scaled: null scale");
    }
    return sharded_planes(g, streams, count, pics, desc, opacity, "glava_b200_sharded_overlay_scaled", scale);
}

int glava_b200_sharded_textures(glava_b200_sharded* g, uint16_t* out_l, uint16_t* out_r) {
    clear_error();
    if (!g) return fail(GLAVA_B200_EINVAL, "null argument");
    return broadcast(g, [=](Shard& s) {
        const size_t n = (size_t) glava_b200_spectrum_size(s.r);
        return glava_b200_textures(s.r, out_l ? out_l + (size_t) s.first * n : nullptr, out_r ? out_r + (size_t) s.first * n : nullptr);
    });
}

}  // extern "C"
