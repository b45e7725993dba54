// TEST INFRASTRUCTURE — host build of stream_state_core.h (the layout and ring rotation of per-stream state blobs).
//
// Drives the pack / unpack kernels' per-vector work (state_pack_kernel / state_unpack_kernel, stream_state_kernels.cu) for
// one stream on host arrays laid out as the renderer's, so the CPU tier can check the blob layout and the average ring's
// age order against a numpy restatement.  Compiled by tests/test_stream_state.py; NOT part of libglava_b200.so.
#include "../../glava_b200/csrc/stream_state_core.h"

#include <cstring>

using namespace glb;

// ptrs = {gravity, ring, spec, tex, av, fifo_l, fifo_r}
static StatePtrs emul_state_ptrs(char* const* ptrs) {
    StatePtrs P;
    P.gravity = ptrs[0]; P.ring = ptrs[1]; P.spec = ptrs[2]; P.tex = ptrs[3]; P.av = ptrs[4]; P.fifo[0] = ptrs[5]; P.fifo[1] = ptrs[6];
    return P;
}

extern "C" {

size_t emul_state_segment_bytes(const StateLayout* L) { return ss_segment_bytes(*L); }

// blob = the segments of stream `stream` (no header), ring rotated out of `cursor`
void emul_state_pack(const StateLayout* L, char* const* ptrs, int stream, uint32_t cursor, char* blob) {
    const StatePtrs P = emul_state_ptrs(ptrs);
    for (uint32_t v = 0; v < ss_stream_vecs(*L); ++v) memcpy(blob + (size_t) v * 16, ss_addr(*L, P, (size_t) stream, cursor, v), 16);
}

// the segments back into stream `stream`, ring rotated into `cursor`; blob == nullptr zeroes them (reset)
void emul_state_unpack(const StateLayout* L, char* const* ptrs, int stream, uint32_t cursor, const char* blob) {
    const StatePtrs P = emul_state_ptrs(ptrs);
    for (uint32_t v = 0; v < ss_stream_vecs(*L); ++v) {
        char* dst = ss_addr(*L, P, (size_t) stream, cursor, v);
        if (blob) memcpy(dst, blob + (size_t) v * 16, 16); else memset(dst, 0, 16);
    }
}

}  // extern "C"
