// stream_state_kernels.cu — pack / unpack / zero of per-stream state (glava_b200_save_streams, _load_streams,
// _reset_streams in capi.cu).
//
// One launch per chunk of streams.  The chunk's table (int stream[count], then uint32 cursor[count]) reaches the device
// in one small copy; every thread moves 16-byte vectors, flattened over (stream, segment, vector) on grid.x only, so the
// batch size never meets the grid-y limit.  The layout and the average ring's age order are stream_state_core.h.
#include "internal.h"
#include "stream_state_core.h"

#include <cuda_runtime.h>

namespace glb {

// blob-ordered staging [count][stream vectors] <- the renderer's arrays
__global__ void __launch_bounds__(256) state_pack_kernel(StateLayout L, StatePtrs P, const int* __restrict__ table, int count,
                                                        uint4* __restrict__ out) {
    const uint32_t sv = ss_stream_vecs(L), total = (uint32_t) count * sv;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t k = i / sv, v = i - k * sv;
        const int s = __ldg(table + k);
        const uint32_t cur = (uint32_t) __ldg(table + count + k);
        out[i] = *reinterpret_cast<const uint4*>(ss_addr(L, P, (size_t) s, cur, v));
    }
}

// the renderer's arrays <- blob-ordered staging; in == nullptr writes zeros (reset)
__global__ void __launch_bounds__(256) state_unpack_kernel(StateLayout L, StatePtrs P, const int* __restrict__ table, int count,
                                                          const uint4* __restrict__ in) {
    const uint32_t sv = ss_stream_vecs(L), total = (uint32_t) count * sv;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t k = i / sv, v = i - k * sv;
        const int s = __ldg(table + k);
        const uint32_t cur = (uint32_t) __ldg(table + count + k);
        *reinterpret_cast<uint4*>(ss_addr(L, P, (size_t) s, cur, v)) = in ? in[i] : make_uint4(0u, 0u, 0u, 0u);
    }
}

static unsigned state_grid(uint32_t total) {
    const uint32_t blocks = (total + 255u) / 256u;
    return blocks < 132u * 16u ? (blocks ? blocks : 1u) : 132u * 16u;   // grid-stride beyond 16 CTAs per SM of an H100 SXM
}

int launch_state_pack(const StateLayout& L, const StatePtrs& P, const int* d_table, int count, void* d_out, void* stream) {
    const uint32_t total = (uint32_t) count * ss_stream_vecs(L);
    state_pack_kernel<<<state_grid(total), 256, 0, (cudaStream_t) stream>>>(L, P, d_table, count, (uint4*) d_out);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "state pack kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

int launch_state_unpack(const StateLayout& L, const StatePtrs& P, const int* d_table, int count, const void* d_in, void* stream) {
    const uint32_t total = (uint32_t) count * ss_stream_vecs(L);
    state_unpack_kernel<<<state_grid(total), 256, 0, (cudaStream_t) stream>>>(L, P, d_table, count, (const uint4*) d_in);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "state unpack kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

}  // namespace glb
