// stream_state_core.h — layout of one stream's state blob and the rotation of its average ring (host and device).
//
// glava_b200_save_streams / _load_streams / _reset_streams (capi.cu) move the per-stream state a renderer keeps between
// updates through one pack and one unpack kernel (stream_state_kernels.cu).  The blob layout, the age order of the
// average ring and the bounds of each segment live here once, so the kernels, glava_b200_stream_state_bytes and the host
// emulation (tests/emul) share one definition.
//
// One stream's segments, per channel read by the module (two, or one for `wave`), every row a multiple of 16 bytes:
//   gravity store                 n   x esz      (esz = 2: pipeline B's u16 state, 4: pipeline A's float state)
//   average ring, age 0 .. F - 1  F x n x esz    (age 0 = the newest frame, independent of the ring cursor)
//   spec                          n   x 4        (latest chain result, glava_b200_spectrum)
//   texture                       n   x 2        (the half the next raster reads and an unmodified update carries)
//   pre-smoothing texture (d_av)  n   x 2        (re-smoothed by the K5 kernels for an unmodified stream)
//   device FIFO ring              n_in x 4       (current ping-pong half, glava_b200_ingest_fifo / _ingest_float)
// A blob is GLB_STATE_HEADER_BYTES of header (StateHeader) followed by these segments, channel 0 first.
#ifndef GLAVA_B200_STREAM_STATE_CORE_H
#define GLAVA_B200_STREAM_STATE_CORE_H

#include <cstddef>
#include <cstdint>

#ifdef __CUDACC__
#define GLB_SS_HD __host__ __device__ __forceinline__
#else
#define GLB_SS_HD inline
#endif

namespace glb {

#define GLB_STATE_MAGIC 0x54534247u          // "GBST" little-endian
#define GLB_STATE_VERSION 1u
#define GLB_STATE_HEADER_BYTES 4096          // = GLAVA_B200_STATE_HEADER_BYTES (include/glava_b200.h)

// segment kinds of one channel, in blob order (GLB_SEG_RING covers F rows)
enum { GLB_SEG_GRAVITY = 0, GLB_SEG_RING = 1, GLB_SEG_SPEC = 2, GLB_SEG_TEX = 3, GLB_SEG_AV = 4, GLB_SEG_FIFO = 5 };

struct StateLayout {
    int n;        // spectrum entries per channel (setbufsize / setbufscale)
    int n_in;     // FIFO ring floats per channel (setbufsize)
    int F;        // setavgframes
    int esz;      // bytes per gravity / average element: 2 (pipeline B) or 4 (pipeline A)
    int chans;    // channels with state: 2, or 1 for wave
};

// 16-byte vectors of each segment row and of one channel
GLB_SS_HD uint32_t ss_state_vecs(const StateLayout& L) { return (uint32_t) L.n * (uint32_t) L.esz / 16u; }
GLB_SS_HD uint32_t ss_chan_vecs(const StateLayout& L) {
    return (1u + (uint32_t) L.F) * ss_state_vecs(L) + (uint32_t) L.n / 4u + (uint32_t) L.n / 8u + (uint32_t) L.n / 8u + (uint32_t) L.n_in / 4u;
}
GLB_SS_HD uint32_t ss_stream_vecs(const StateLayout& L) { return (uint32_t) L.chans * ss_chan_vecs(L); }
GLB_SS_HD size_t ss_segment_bytes(const StateLayout& L) { return (size_t) ss_stream_vecs(L) * 16u; }
GLB_SS_HD size_t ss_blob_bytes(const StateLayout& L) { return (size_t) GLB_STATE_HEADER_BYTES + ss_segment_bytes(L); }

// Ring slot holding the frame of age `age` (0 = newest) for a stream whose next modified update writes slot `cursor`
// (the spectrum kernels' out_idx: modified updates of that stream so far, mod F).
GLB_SS_HD int ss_ring_slot(int age, uint32_t cursor, int F) {
    int s = (int) cursor - 1 - age;
    s %= F;
    return s < 0 ? s + F : s;
}

// Where 16-byte vector `v` of a stream's segments lives: channel, segment kind, row (the ring age for GLB_SEG_RING, else 0)
// and the vector offset inside that row.
struct SegPos { int ch, kind, row; uint32_t off; };
GLB_SS_HD SegPos ss_locate(const StateLayout& L, uint32_t v) {
    SegPos q;
    const uint32_t cv = ss_chan_vecs(L), sv = ss_state_vecs(L);
    q.ch = (int) (v / cv);
    uint32_t w = v - (uint32_t) q.ch * cv;
    const uint32_t st = (1u + (uint32_t) L.F) * sv;
    q.row = 0;
    if (w < st) {
        const uint32_t r = w / sv;
        q.off = w - r * sv;
        q.kind = r == 0 ? GLB_SEG_GRAVITY : GLB_SEG_RING;
        q.row = r == 0 ? 0 : (int) r - 1;
        return q;
    }
    w -= st;
    if (w < (uint32_t) L.n / 4u) { q.kind = GLB_SEG_SPEC; q.off = w; return q; }
    w -= (uint32_t) L.n / 4u;
    if (w < (uint32_t) L.n / 8u) { q.kind = GLB_SEG_TEX; q.off = w; return q; }
    w -= (uint32_t) L.n / 8u;
    if (w < (uint32_t) L.n / 8u) { q.kind = GLB_SEG_AV; q.off = w; return q; }
    w -= (uint32_t) L.n / 8u;
    q.kind = GLB_SEG_FIFO; q.off = w;
    return q;
}

// Base pointers of a renderer's state arrays (device pointers in the kernels, host arrays in the emulation).
//   gravity [batch*2][n] x esz, ring [batch*2][F][n] x esz, spec [batch*2][n] f32, tex / av [batch*2][n] u16,
//   fifo[ch] [batch][n_in] f32
struct StatePtrs {
    char* gravity; char* ring; char* spec; char* tex; char* av; char* fifo[2];
};

// Address of vector `v` of stream `s` (ring cursor `cursor`) in the renderer's arrays
GLB_SS_HD char* ss_addr(const StateLayout& L, const StatePtrs& P, size_t s, uint32_t cursor, uint32_t v) {
    const SegPos q = ss_locate(L, v);
    const size_t plane = s * 2 + (size_t) q.ch, n = (size_t) L.n, off = (size_t) q.off * 16u;
    switch (q.kind) {
    case GLB_SEG_GRAVITY: return P.gravity + plane * n * (size_t) L.esz + off;
    case GLB_SEG_RING:
        return P.ring + (plane * (size_t) L.F + (size_t) ss_ring_slot(q.row, cursor, L.F)) * n * (size_t) L.esz + off;
    case GLB_SEG_SPEC: return P.spec + plane * n * 4u + off;
    case GLB_SEG_TEX: return P.tex + plane * n * 2u + off;
    case GLB_SEG_AV: return P.av + plane * n * 2u + off;
    default: return (q.ch ? P.fifo[1] : P.fifo[0]) + s * (size_t) L.n_in * 4u + off;   // (no dynamic index: keeps P out of local memory)
    }
}

// The fixed part of a blob's header (zero-padded to GLB_STATE_HEADER_BYTES); `params` is the source's effective
// glava_b200_params (setbufsize / setbufscale, accel_fft as the kernels run it) with fb_slots zeroed, stored as raw bytes.
struct StateHeader {
    uint32_t magic, version, header_bytes, params_bytes;
    uint64_t blob_bytes;
    uint64_t reserved;
};

}  // namespace glb

#endif
