// spectrum_kernels.cu — sm_90a kernels of the PCM -> R16 texture half of the path.
//
//   spectrum_kernel    one work unit per (stream, channel): TMA bulk load of the PCM ring into shared memory,
//                      window, (N/2)-point Stockham FFT in shared memory, |.|/log/ramp, gravity + average
//                      (pipeline A float state or pipeline B R16 state in HBM), lazy K5 smoothing out of
//                      shared memory -> R16 texture.   [replaces render.c transform_fft/gravity/average +
//                      util/{pass,gravity_pass,average_pass,smooth_pass}.frag + 5 GL draws and one
//                      glTexImage1D per channel per frame]
//   k5_planes_kernel   K5 for whole planes, tap weights shared between 8 planes
//   fifo_ingest_kernel fifo.c:89-110 on the device-resident rings
//
// Compiled with --fmad=false: results are bit-identical to the host build of the *_core.h maths.
#include "internal.h"
#include "raster_core.h"
#include "spectrum_plan.h"

#include <cuda_runtime.h>

#include <type_traits>

namespace glb {

// ---------------------------------------------------------------------------------------------
// small PTX wrappers: mbarrier + 1-D bulk async copy (TMA engine, SASS UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n .reg .pred p;\n WAIT_%=:\n"
        " mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        " @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// grid.y is limited to 65535 and a batch is not (glava_b200_new takes any batch >= 1): a launcher whose y axis counts planes,
// streams or groups of planes launches slices of at most that many rows, each told its first row (launch_raster chunks its
// batch axis the same way).  `launch(y0, rows)` enqueues one slice.
constexpr int GRID_Y_MAX = 65535;
template <class Launch>
static cudaError_t launch_y_slices(int rows, Launch launch) {
    for (int y0 = 0; y0 < rows; y0 += GRID_Y_MAX) {
        launch(y0, (unsigned) min(GRID_Y_MAX, rows - y0));
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------
// spectrum kernel
constexpr int spec_default_threads(int log2n) {
    const int m8 = (1 << log2n) / 16;
    return m8 < 128 ? 128 : (m8 > 512 ? 512 : m8);
}
// OOP = out-of-place passes between two buffers: one barrier per pass instead of two and a thread holds ONE butterfly in
// registers at a time (in place it must hold all of its butterflies across the barrier: 116-124 registers at N >= 8192,
// one 512-thread CTA per SM).  With half the registers and small CTAs several planes are resident per SM, their barrier
// waits overlap, and the kernel co-resides with the raster kernel's CTAs instead of alternating with them.
template <int LOG2N, int TT = 0, bool OOP = false> struct SpecCfg {
    static constexpr int N = 1 << LOG2N, M = N / 2;
    static constexpr int T = TT > 0 ? TT : spec_default_threads(LOG2N);
    static constexpr int BUF_BYTES = spectrum_buf_bytes(N);
    // in place:     cpx buffer (also the raw-PCM staging area, N floats = M cpx) | u16 av[N] | mbarriers (spectrum_plan.h)
    // out of place: buffer A (PCM lands here) | buffer B | mbarriers; av[N] lives in whichever buffer the result is NOT in
    static constexpr int OFF_B   = BUF_BYTES;
    static constexpr int OFF_AV  = BUF_BYTES;
    static constexpr int SMEM    = OOP ? 2 * BUF_BYTES + 16 : spectrum_smem_bytes(N);
    static constexpr int OFF_BAR = SMEM - 16;
    static constexpr bool RESULT_IN_B = OOP && (fft_pass_count(M) % 2 == 1);
    // Twiddle table (M complex floats) in shared memory, behind the mbarriers, landed by the TMA engine with the CTA's first
    // PCM load: in place up to N = 4096 (16 KB there), where it fits beside the buffers at the size's residency and a
    // thread's first pass is one butterfly (its window factors are prefetched before the PCM wait).  At 8192 (out of place,
    // 3 CTAs/SM by shared memory) the table would cost a resident CTA, at 16384 a thread holds two first-pass butterflies:
    // there the passes read the table through L1.
    static constexpr bool TW_SMEM  = !OOP && N <= 4096;
    static constexpr int  TW_BYTES = TW_SMEM ? M * 8 : 0;
    static constexpr int  OFF_TW   = SMEM;
    // fixed dynamic shared memory of the FFT (twiddles) or wave kernel; the K5 tap table follows it
    static constexpr int  dyn_bytes(bool is_fft) { return SMEM + (is_fft ? TW_BYTES : 0); }
    static constexpr int  R0 = M >= 8 ? 8 : M, NB0 = M / R0;   // first pass: radix, butterflies (fft_core.h, NS = 1)
    static_assert(!TW_SMEM || NB0 <= T, "shared-memory twiddle form: one first-pass butterfly per thread");
    // resident CTAs per SM the register allocation must allow: the kernel waits on memory a lot (TMA load,
    // state loads), so occupancy is worth more than the last registers (128 regs -> 2 CTAs/SM was measured)
    static constexpr int SMEM_CTAS = (220 * 1024) / SMEM < 1 ? 1 : (220 * 1024) / SMEM;
    static constexpr int OOP_CTAS  = (1024 / T) < SMEM_CTAS ? (1024 / T) : SMEM_CTAS;       // (T = 1024: 1)       // <= 64 registers where shared memory allows
    static constexpr int MIN_CTAS = OOP ? (OOP_CTAS < 1 ? 1 : OOP_CTAS)
                                        : (T >= 512 ? 1 : (T * (N / 16 / T > 1 ? 2 : 1) > 256 ? 2 : 3));   // T = 512: capping at 64 registers spills in the FFT passes and was measured slower
};

template <int M, int T, int NS, class Loader>
__device__ __forceinline__ void run_passes(cpx* buf, Loader first_loader, const cpx* __restrict__ tw, int tid) {
    constexpr int REM = M / NS;                      // points still to be combined
    if constexpr (REM > 1) {
        constexpr int R = (REM >= 8) ? 8 : REM;      // 8, 8, ..., then 4 or 2
        using Pass = StockhamPass<M, T, R, NS>;
        cpx reg[Pass::PER][R];
        if constexpr (NS == 1) Pass::load(first_loader, tw, tid, reg);
        else Pass::load([buf](int i) { return buf[fft_pad(i)]; }, tw, tid, reg);
        __syncthreads();
        Pass::store(buf, tid, reg);
        __syncthreads();
        run_passes<M, T, NS * R>(buf, first_loader, tw, tid);
    }
}
// out of place: src -> dst, one barrier, then the roles swap (the first pass reads the raw PCM through `first_loader`)
template <int M, int T, int NS, class Loader>
__device__ __forceinline__ void run_passes_oop(cpx* src, cpx* dst, Loader first_loader, const cpx* __restrict__ tw, int tid) {
    constexpr int REM = M / NS;
    if constexpr (REM > 1) {
        constexpr int R = (REM >= 8) ? 8 : REM;
        using B = StockhamButterfly<M, R, NS>;
        auto st = [dst](int i, cpx v) { dst[fft_pad(i)] = v; };
        for (int j = tid; j < B::NB; j += T) {
            if constexpr (NS == 1) B::run(j, first_loader, st, tw);
            else B::run(j, [src](int i) { return src[fft_pad(i)]; }, st, tw);
        }
        __syncthreads();
        run_passes_oop<M, T, NS * R>(dst, src, first_loader, tw, tid);
    }
}

extern __shared__ __align__(16) unsigned char glb_smem[];

template <int LOG2N, bool IS_FFT, int TT = 0, bool OOP = false>
__global__ void __launch_bounds__((SpecCfg<LOG2N, TT, OOP>::T), (SpecCfg<LOG2N, TT, OOP>::MIN_CTAS))
spectrum_kernel(const __grid_constant__ SpectrumArgs a, const __grid_constant__ glava_b200_params p) {
    using C = SpecCfg<LOG2N, TT, OOP>;
    constexpr int N = C::N, M = C::M, T = C::T;
    const int tid = threadIdx.x;

    // buf = where the transform's result is read from; av = the R16 texels of the epilogue (out of place: in the other buffer)
    cpx*      bufA = reinterpret_cast<cpx*>(glb_smem);
    cpx*      bufB = reinterpret_cast<cpx*>(glb_smem + C::OFF_B);
    cpx*      buf = (OOP && C::RESULT_IN_B) ? bufB : bufA;
    float*    raw = reinterpret_cast<float*>(glb_smem);
    uint16_t* av  = OOP ? reinterpret_cast<uint16_t*>((IS_FFT && C::RESULT_IN_B) ? bufA : bufB) : reinterpret_cast<uint16_t*>(glb_smem + C::OFF_AV);
    uint64_t* bar = reinterpret_cast<uint64_t*>(glb_smem + C::OFF_BAR);
    cpx*      twsm = reinterpret_cast<cpx*>(glb_smem + C::OFF_TW);
    const cpx* const tw = C::TW_SMEM ? twsm : reinterpret_cast<const cpx*>(a.twiddle);

    // Persistent CTAs: work unit u = one (stream, channel) plane (wave: one stream, audio_l only,
    // wave/1.frag:7); a CTA walks u = blockIdx.x, + gridDim.x, ...  The PCM ring of the NEXT unit is
    // prefetched by the TMA engine while this unit's smoothing pass runs.
    const int units = IS_FFT ? a.batch * 2 : a.batch;
    // one bulk async copy, N*4 bytes, completes on `bar`; the CTA's first one also lands the twiddle table
    auto issue_load = [&](int u, bool with_tw = false) {
        const int cc = IS_FFT ? u : 2 * u;
        const float* pcm = ((cc & 1) == 0 ? a.pcm_l : a.pcm_r) + (size_t) (cc >> 1) * N;
        // the buffer was last touched through the generic proxy (FFT passes): order those accesses
        // before the async-proxy (TMA) write
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(bar, N * 4 + (with_tw ? C::TW_BYTES : 0));
        bulk_g2s(raw, pcm, N * 4, bar);
        if (with_tw) bulk_g2s(twsm, a.twiddle, C::TW_BYTES, bar);
    };
    // K5 tap table of this CTA's channel in shared memory (behind the fixed regions): one more bulk copy, in flight
    // during the FFT and the epilogue
    unsigned char* tapsm = glb_smem + C::dyn_bytes(IS_FFT);
    uint64_t* bar2 = bar + 1;
    auto issue_tab = [&](int ch) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(bar2, (uint32_t) a.csr_bytes);
        const unsigned char* src = a.csr + (size_t) ch * a.csr_bytes;
        for (int o = 0; o < a.csr_bytes; o += 32768)
            bulk_g2s(tapsm + o, src + o, (uint32_t) min(32768, a.csr_bytes - o), bar2);
    };
    if (tid == 0) { mbar_init(bar, 1); mbar_init(bar2, 1); }
    __syncthreads();
    if (tid == 0 && (int) blockIdx.x < units) issue_load(blockIdx.x, IS_FFT && C::TW_SMEM);
    int tab_ch = -1; bool tab_pending = false; uint32_t parity2 = 0;
    if (a.csr && a.need && (int) blockIdx.x < units && !a.skip_tex && p.smooth_pass) {
        tab_ch = IS_FFT ? ((int) blockIdx.x & 1) : 0;
        if (tid == 0) issue_tab(tab_ch);
        tab_pending = true;
    }
    uint32_t parity = 0;
    const int F = p.avg_frames;

  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int c = IS_FFT ? u : 2 * u, ch = c & 1;
    const size_t plane = (size_t) c * N;
    // per-stream `modified` (glava.c:528-537, render.c:2268-2272): a stream without new audio keeps its gravity / average
    // state and shows its previous texture again
    const uint32_t um = a.umask ? __ldg(a.umask + (c >> 1)) : 0x80000000u;
    const int cursor = a.umask ? (int) (um & 0xffffu) : (int) (a.update % (unsigned long long) F);
    if (!(um >> 31)) {
        mbar_wait(bar, parity); parity ^= 1u;        // (the prefetched ring is not used)
        if (!a.skip_tex && a.tex_prev) {
            const uint4* src = reinterpret_cast<const uint4*>(a.tex_prev + plane);
            uint4* dst = reinterpret_cast<uint4*>(a.tex + plane);
            for (int i = tid; i < N / 8; i += T) dst[i] = src[i];
        }
        __syncthreads();
        if (tid == 0 && u + (int) gridDim.x < units) issue_load(u + gridDim.x);
        continue;
    }
    if (IS_FFT && p.accel_fft && !a.fft_only) {
        // while the PCM load is in flight: pull the R16 state the pipeline-B epilogue below reads (HBM-resident) towards L2,
        // so its loads after the FFT are L2 hits: the leading bins it runs over of the gravity plane (s = 0) and of the F - 1
        // ring slots it averages (s = 1 .. F-1: slot cursor - s).  Not the slot it overwrites, nothing past its bins.  (The
        // FFT-only form reads no state: epilogue_b_kernel does, after the whole grid.)
        // (the epilogue rounds epi_n up to a multiple of T: those last few bins are not prefetched)
        const int lines = (a.epi_n > 0 && a.epi_n < N) ? (a.epi_n * 2 + 127) / 128 : (N * 2) / 128;
        const char* g0 = reinterpret_cast<const char*>(a.gr_store + plane);
        const char* r0 = reinterpret_cast<const char*>(a.ring_u + plane * F);
        for (int s = 0; s < F; ++s) {
            int fr = cursor - s; if (fr < 0) fr += F;
            const char* src = s == 0 ? g0 : r0 + (size_t) fr * N * 2;
            for (int l = tid; l < lines; l += T) asm volatile("prefetch.global.L2 [%0];" ::"l"(src + (size_t) l * 128));
        }
    }
    if constexpr (IS_FFT && C::TW_SMEM) {
        // the window factors of this thread's first-pass butterfly (j = tid: points tid + t * NB0) towards L1 before the
        // wait, so that their L2 latency overlaps the TMA.  (Held in registers instead, 32 of them, they spill under the
        // 3-CTA register cap at 4096.)
        if (tid < C::NB0) {
#pragma unroll
            for (int t = 0; t < C::R0; ++t)
                asm volatile("prefetch.global.L1 [%0];" ::"l"(reinterpret_cast<const double2*>(a.window) + tid + t * C::NB0));
        }
    }
    mbar_wait(bar, parity); parity ^= 1u;

    if constexpr (IS_FFT) {
        // --- window (render.c:793-795: float * double -> float) folded into the first pass loads ----
        const double2* w2 = reinterpret_cast<const double2*>(a.window);
        auto first = [raw, w2](int i) {
            float2 v = reinterpret_cast<const float2*>(raw)[i];
            double2 w = __ldg(&w2[i]);
            cpx r = { (float) ((double) v.x * w.x), (float) ((double) v.y * w.y) };
            return r;
        };
        if constexpr (OOP) run_passes_oop<M, T, 1>(bufA, bufB, first, tw, tid);
        else run_passes<M, T, 1>(buf, first, tw, tid);

        if (a.fft_only) {
            // transform_fft's tail only (render.c:842-846); the state update and K5 follow as full-occupancy kernels
            const int lim = (a.epi_n > 0 && a.epi_n < N) ? a.epi_n : N;
            float* const spec = a.spec + plane;
            for (int n = tid; n < lim; n += T) {
                cpx z = buf[fft_pad(n >> 1)];
                spec[n] = fft_post((n & 1) ? z.y : z.x, n, N, p.fft_scale, p.fft_cutoff);
            }
            __syncthreads();
            if (tid == 0 && u + (int) gridDim.x < units) issue_load(u + gridDim.x);
            continue;
        }
        if (!p.accel_fft) {
            // --- pipeline A: render.c:2149-2156 --------------------------------------------------
            const float g = p.gravity_step * (1.0f / p.ur);
            const int newest = cursor;
            for (int n = tid; n < N; n += T) {
                cpx z = buf[fft_pad(n >> 1)];
                float v = fft_post((n & 1) ? z.y : z.x, n, N, p.fft_scale, p.fft_cutoff);
                v = gravity_a(v, &a.applied[plane + n], g);
                float* ring = a.ring_f + plane * F;
                ring[(size_t) newest * N + n] = v;
                float acc = 0.0f;
                for (int f = 0; f < F; ++f) {                      // oldest first, like the memmove'd ring
                    int slot = newest + 1 + f; if (slot >= F) slot -= F;
                    float b = (f == F - 1) ? v : ring[(size_t) slot * N + n];
                    if (p.avg_window) acc = (float) ((double) acc + a.avg_w_a[f] * (double) b);
                    else acc += b;
                }
                float out = acc / (float) F;
                a.spec[plane + n] = out;
                av[n] = (uint16_t) unorm16(out);                   // glTexImage1D GL_R16 upload, render.c:521-524
            }
        } else {
            // --- pipeline B: render.c:2177-2267 ---------------------------------------------------
            const float diff = p.gravity_step * (1.0f / p.ur);
            const int out_idx = cursor;
            const int epi_n = (a.epi_n > 0 && a.epi_n < N) ? ((a.epi_n + T - 1) / T) * T : N;
            float*    const spec = a.spec + plane;
            uint16_t* const grs  = a.gr_store + plane;
            uint16_t* const ring = a.ring_u + plane * F;
            // FT = compile-time copy of F for the common small values: the slot offsets and the
            // weights of the average live in registers and the tap loop is fully unrolled
            auto epilogue = [&](auto ft) {
                constexpr int FT = decltype(ft)::value;               // 0 = generic (runtime F)
                const int FF = FT ? FT : F;
                int off[FT ? FT : 1]; float wt[FT ? FT : 1];
                if constexpr (FT > 0) {
#pragma unroll
                    for (int i = 0; i < FT; ++i) {
                        int fr = out_idx - i; if (fr < 0) fr += FT;
                        off[i] = fr * N; wt[i] = a.avg_w_b[i];
                    }
                }
                if constexpr (FT > 0) {
                    // 4 elements per trip: all their state loads (1 + FT-1 each) are issued before the
                    // first dependent use, so the global-load latency is paid once per trip, not per element
                    constexpr int U = (N / T) % 2 == 0 ? 2 : 1;   // 4 was measured to cost registers (spills under the occupancy cap) for no gain
                    static_assert((N / T) % U == 0, "N / T must be a multiple of the epilogue unroll");
                    // epi_n (multiple of T): with lazy K5 only the leading bins that some sampled texel's
                    // taps can reach are post-processed (their state is all that can influence a pixel)
                    for (int n0 = tid; n0 < epi_n; n0 += U * T) {
                        uint32_t g_old[U], rg[U][FT];
#pragma unroll
                        for (int e = 0; e < U; ++e) {
                            const int n = n0 + e * T;
                            if (n >= epi_n) continue;
                            g_old[e] = grs[n];
#pragma unroll
                            for (int i = 1; i < FT; ++i) rg[e][i] = ring[off[i] + n];
                        }
#pragma unroll
                        for (int e = 0; e < U; ++e) {
                            const int n = n0 + e * T;
                            if (n >= epi_n) continue;
                            cpx z = buf[fft_pad(n >> 1)];
                            float v = fft_post((n & 1) ? z.y : z.x, n, N, p.fft_scale, p.fft_cutoff);
                            spec[n] = v;
                            uint32_t gq = gravity_b(unorm16(v), g_old[e], diff);
                            grs[n] = (uint16_t) gq;
                            uint32_t texel = gq;
                            if (FT > 1) {
                                ring[off[0] + n] = (uint16_t) gq;
                                float r = 0.0f;
#pragma unroll
                                for (int i = 0; i < FT; ++i) {         // t0 = most recent (render.c:2250-2255)
                                    float tx = from16(i == 0 ? gq : rg[e][i]);
                                    if (a.avg_b_windowed) r += wt[i] * tx; else r += tx;
                                }
                                texel = unorm16(r / (float) FT);
                            }
                            av[n] = (uint16_t) texel;
                        }
                    }
                } else {
                    for (int n = tid; n < epi_n; n += T) {             // any F: runtime loop
                        cpx z = buf[fft_pad(n >> 1)];
                        float v = fft_post((n & 1) ? z.y : z.x, n, N, p.fft_scale, p.fft_cutoff);
                        spec[n] = v;
                        uint32_t gq = gravity_b(unorm16(v), grs[n], diff);
                        grs[n] = (uint16_t) gq;
                        uint32_t texel = gq;
                        if (FF > 1) {
                            float r = 0.0f;
                            ring[(size_t) out_idx * N + n] = (uint16_t) gq;
                            for (int i = 0; i < F; ++i) {
                                int fr = out_idx - i; if (fr < 0) fr += F;
                                float tx = from16(i == 0 ? gq : (uint32_t) ring[(size_t) fr * N + n]);
                                if (a.avg_b_windowed) r += a.avg_w_b[i] * tx; else r += tx;
                            }
                            texel = unorm16(r / (float) FF);
                        }
                        av[n] = (uint16_t) texel;
                    }
                }
            };
            switch (F) {
                case 5: epilogue(std::integral_constant<int, 5>()); break;       // shipped default (smooth_parameters.glsl:56)
                case 6: epilogue(std::integral_constant<int, 6>()); break;       // compiled-in default (render.c:912)
                case 3: epilogue(std::integral_constant<int, 3>()); break;
                case 4: epilogue(std::integral_constant<int, 4>()); break;
                default: epilogue(std::integral_constant<int, 0>()); break;
            }
        }
    } else {
        // --- wave: "window" (no-op) + "wrange" (render.c:773-781), upload ---------------------------
        for (int n = tid; n < N; n += T) {
            float b = raw[n];
            b += 1.0f; b /= 2.0f;
            a.spec[plane + n] = b;
            av[n] = (uint16_t) unorm16(b);
        }
    }
    __syncthreads();
    // `raw`/`buf` are dead from here on: let the TMA engine fetch the next unit's PCM during K5 (out of place, `av` may live
    // in the landing buffer: the load is issued after K5)
    if (!OOP && tid == 0 && u + (int) gridDim.x < units) issue_load(u + gridDim.x);
    if (a.skip_tex) { if (OOP && tid == 0 && u + (int) gridDim.x < units) issue_load(u + gridDim.x); continue; }   // chain result only (`spec`): the texture is produced downstream

    // --- K5 smooth pass out of shared memory (render.c:2276-2303) ----------------------------------
    uint16_t* tex = a.tex + plane;
    if (p.smooth_pass) {
        const SmoothParams sp = smooth_params(p);
        if (a.need && a.csr) {
            // taps from shared memory: per tap two LDS + the texel fetch, no global-memory latency on the serial sum
            if (tab_ch != ch) {                      // persistent CTA whose unit changed channel (odd grid): reload
                if (tid == 0) issue_tab(ch);
                tab_ch = ch; tab_pending = true;
            }
            if (tab_pending) { mbar_wait(bar2, parity2); parity2 ^= 1u; tab_pending = false; }
            const float*    tw = reinterpret_cast<const float*>(tapsm);
            const uint16_t* ti = reinterpret_cast<const uint16_t*>(tapsm + a.csr_idx_off);
            const int*      to = reinterpret_cast<const int*>(tapsm + a.csr_off_off);
            const int* need = a.need + (size_t) ch * a.need_count;
            for (int k = tid; k < a.need_count; k += T) {
                const int x = need[k];
                if (x < 0 || x >= N) continue;
                const int o0 = to[k], o1 = to[k + 1];
                SmoothAcc acc; acc.init();
                // the sum is serial in the tap order (smooth.glsl:33-37), but its operands are not: fetch KU taps' index,
                // weight and texel (two dependent shared-memory round trips) before the KU dependent adds
                constexpr int KU = 8;
                int o = o0;
                for (; o + KU <= o1; o += KU) {
                    int ii[KU]; float ww[KU], tx[KU];
#pragma unroll
                    for (int q = 0; q < KU; ++q) { ii[q] = ti[o + q]; ww[q] = tw[o + q]; }
#pragma unroll
                    for (int q = 0; q < KU; ++q) tx[q] = from16(av[ii[q]]);      // (a tap outside the texture is stored as index 0, weight 0)
#pragma unroll
                    for (int q = 0; q < KU; ++q) acc.add_noweight(tx[q], ww[q]);
                }
                for (; o < o1; ++o) {
                    acc.add_noweight(from16(av[ti[o]]), tw[o]);
                }
                acc.weight = a.tap_wsum[(size_t) ch * a.need_count + k];
                tex[x] = (uint16_t) unorm16(acc.result(sp));
            }
        } else if (a.need && a.tap_tab) {
            // weights / indices precomputed once (they depend on the parameters only): per tap one
            // coalesced 8-byte load, one shared-memory texel fetch, a multiply and an add
            const int* need = a.need + (size_t) ch * a.need_count;
            const TapEntry* tab = a.tap_tab + (size_t) ch * a.tap_max * a.need_count;
            // a thread's taps are a serial float sum, but the table loads are independent of it: fetch KU entries (one
            // L2 round trip) before consuming them, in the GLSL loop's order.  (A tap outside the texture is stored as
            // index 0 / weight 0: no range test on the chain.)
            auto sums = [&](auto ku_tag) {
                constexpr int KU = decltype(ku_tag)::value;
                for (int k = tid; k < a.need_count; k += T) {
                    const int x = need[k];
                    if (x < 0 || x >= N) continue;
                    const int cnt = a.tap_cnt[(size_t) ch * a.need_count + k];
                    SmoothAcc acc; acc.init();
                    const int2* col = reinterpret_cast<const int2*>(tab) + k;
                    int j = 0;
                    for (; j + KU <= cnt; j += KU) {
                        int2 e[KU];
#pragma unroll
                        for (int q = 0; q < KU; ++q) e[q] = __ldg(col + (size_t) (j + q) * a.need_count);
#pragma unroll
                        for (int q = 0; q < KU; ++q) acc.add_noweight(from16(av[e[q].x]), __int_as_float(e[q].y));
                    }
                    for (; j < cnt; ++j) {
                        const int2 e = __ldg(col + (size_t) j * a.need_count);
                        acc.add_noweight(from16(av[e.x]), __int_as_float(e.y));
                    }
                    acc.weight = a.tap_wsum[(size_t) ch * a.need_count + k];
                    tex[x] = (uint16_t) unorm16(acc.result(sp));
                }
            };
            if (a.tap_ku >= 8) sums(std::integral_constant<int, 8>());
            else if (a.tap_ku >= 4) sums(std::integral_constant<int, 4>());
            else sums(std::integral_constant<int, 2>());
        } else if (a.need) {
            const int* need = a.need + (size_t) ch * a.need_count;
            for (int k = tid; k < a.need_count; k += T) {
                int x = need[k];
                if (x >= 0 && x < N) tex[x] = (uint16_t) smooth_pass_texel(sp, av, N, x);
            }
        } else if (a.av_out) {
            // export the pre-smoothing texture for a K5 kernel downstream: all n texels (k5_table_kernel / k5_planes_kernel
            // smooth whole planes, sharing every tap weight between several planes), or only the leading av_t_len bins the
            // need-list's taps can reach (k5_need_smem_kernel, or av_transpose_kernel + k5_need_kernel)
            uint16_t* dst = a.av_out + plane;
            const int lim = a.av_t_len > 0 ? a.av_t_len : N;
            for (int x = tid; x < lim; x += T) dst[x] = av[x];
        } else {
            for (int x = tid; x < N; x += T) tex[x] = (uint16_t) smooth_pass_texel(sp, av, N, x);
        }
    } else {
        for (int x = tid; x < N; x += T) tex[x] = av[x];
    }
    __syncthreads();                                 // `av` may be overwritten by the next unit's epilogue
    if (OOP && tid == 0 && u + (int) gridDim.x < units) issue_load(u + gridDim.x);
  }
  if (tab_pending) mbar_wait(bar2, parity2);          // (every unit of this CTA was skipped: do not exit under an in-flight bulk copy)
}

int spectrum_threads(int n) {
    switch (n) {
        case 256:   return SpecCfg<8>::T;   case 512:   return SpecCfg<9>::T;
        case 1024:  return SpecCfg<10>::T;  case 2048:  return SpecCfg<11>::T;
        case 4096:  return SpecCfg<12>::T;  case 8192:  return SpecCfg<13>::T;
        case 16384: return SpecCfg<14>::T;  default: return -1;
    }
}
template <int LOG2N, bool IS_FFT, int TT = 0, bool OOP = false>
static int launch_spectrum_t(const glava_b200_params& p, const SpectrumArgs& a, int grid, int resident, cudaStream_t st) {
    using C = SpecCfg<LOG2N, TT, OOP>;
    auto kern = spectrum_kernel<LOG2N, IS_FFT, TT, OOP>;
    // Residency cap (tuning aid, off): the kernel co-runs with the raster kernel (capi.cu run_update) and
    // at full occupancy (5 CTAs x 256 threads x 48 registers per SM) takes most of the register file.
    // Requesting more dynamic shared memory than needed caps it at `resident` CTAs per SM; off, because the
    // stretched spectrum kernel (and the L1 it takes from the raster kernel) costs more than it frees.
    int smem_req = C::dyn_bytes(IS_FFT) + (a.csr ? a.csr_bytes : 0);   // + the K5 tap table of one channel (shared-memory K5 path)
    if (resident > 0) { int want = (227 * 1024) / resident - 1024; if (want > smem_req) smem_req = want; }
    if (smem_req > 227 * 1024) smem_req = 227 * 1024;
    if (smem_req > 48 * 1024) {
        // per-device function attribute: set on every launch (handles on several devices may live in one process)
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_req);
        if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "cudaFuncSetAttribute(spectrum): %s", cudaGetErrorString(e));
    }
    kern<<<grid, C::T, smem_req, st>>>(a, p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "spectrum kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// Variant selection (spectrum_plan.h): default = the measured-best one per size; GLAVA_B200_SPEC_OOP=0|1 and
// GLAVA_B200_SPEC_T=128|256|512 override it for tuning sweeps (tools/spec_probe.py).
template <int L>
static int launch_spectrum_fft(const glava_b200_params& p, const SpectrumArgs& a, int grid, int resident, cudaStream_t st,
                               int oop, int tsel) {
    if (oop) {
        if (tsel == 128) return launch_spectrum_t<L, true, 128, true>(p, a, grid, resident, st);
        if (tsel == 512) { if constexpr (L >= 13) return launch_spectrum_t<L, true, 512, true>(p, a, grid, resident, st); }
        if (tsel == 1024) { if constexpr (L >= 14) return launch_spectrum_t<L, true, 1024, true>(p, a, grid, resident, st); }
        return launch_spectrum_t<L, true, 256, true>(p, a, grid, resident, st);
    }
    if (tsel == 256) { if constexpr (L >= 13) return launch_spectrum_t<L, true, 256, false>(p, a, grid, resident, st); }
    return launch_spectrum_t<L, true, 0, false>(p, a, grid, resident, st);
}

static int launch_spectrum(const glava_b200_params& p, const SpectrumPlan& pl, const SpectrumArgs& a, cudaStream_t st) {
    const bool is_fft = p.module != GLAVA_B200_MOD_WAVE;
    const int grid = pl.spec_grid, resident = pl.spec_resident;
    const int tsel = a.variant_t, oop = a.variant_oop;
#define GLB_CASE(L) case (1 << L): return is_fft ? launch_spectrum_fft<L>(p, a, grid, resident, st, oop, tsel) \
                                                 : launch_spectrum_t<L, false>(p, a, grid, resident, st);
    switch (p.n) {
        GLB_CASE(8) GLB_CASE(9) GLB_CASE(10) GLB_CASE(11) GLB_CASE(12) GLB_CASE(13) GLB_CASE(14)
        default: return fail(GLAVA_B200_EINVAL, "unsupported setbufsize %d", p.n);
    }
#undef GLB_CASE
}

// K5 for whole planes (all n output texels): util/smooth_pass.frag over `count` R16 planes.
// The tap indices and weights of an output texel depend on the parameters only, so one thread computes
// them once (the expensive part: log, divide, sine) and applies them to K5_S planes held in shared
// memory; per plane and tap only a fetch, a multiply and an add remain.  Per-plane arithmetic and
// summation order are exactly smooth_audio()'s.
#define K5_S  8
#define K5_XT 128
__global__ void __launch_bounds__(K5_XT)
k5_planes_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, int n, int count,
                 const __grid_constant__ glava_b200_params p, int y0) {
    uint16_t* seg = reinterpret_cast<uint16_t*>(glb_smem);           // [K5_S][span]
    const SmoothParams sp = smooth_params(p);
    const int x0 = blockIdx.x * K5_XT, x1 = min(n, x0 + K5_XT);
    const int pl0 = (y0 + (int) blockIdx.y) * K5_S, npl = min(K5_S, count - pl0);
    // input index range any tap of this block's texels can touch (scale_audio is increasing)
    const float fn = (float) n;
    const float lo_f = scale_audio(sp, g_clamp(((float) x0 + 0.5f) / fn - sp.smooth_factor, 0.0f, 1.0f)) * fn;
    const float hi_f = scale_audio(sp, g_clamp(((float) (x1 - 1) + 0.5f) / fn + sp.smooth_factor, 0.0f, 1.0f)) * fn;
    int lo = (int) floorf(lo_f) - 2, hi = (int) ceilf(hi_f) + 3;
    lo = lo < 0 ? 0 : lo; hi = hi > n ? n : hi;
    const int span = hi > lo ? hi - lo : 0;
    for (int i = threadIdx.x; i < npl * span; i += K5_XT) {
        const int pl = i / span, k = i - pl * span;
        seg[pl * span + k] = in[(size_t) (pl0 + pl) * n + lo + k];
    }
    __syncthreads();
    const int x = x0 + threadIdx.x;
    if (x >= x1) return;
    SmoothAcc acc[K5_S];
#pragma unroll
    for (int s = 0; s < K5_S; ++s) acc[s].init();
    smooth_enumerate(sp, n, ((float) x + 0.5f) / fn, [&](int i, float w) {
        const int k = i - lo;
        const bool valid = (i >= 0 && i < n);                          // outside [0, n): texelFetch reads 0
        const bool staged = valid && k >= 0 && k < span;               // (always, unless the range estimate is off)
#pragma unroll
        for (int s = 0; s < K5_S; ++s) {
            float texel = 0.0f;
            if (valid && s < npl) texel = from16(staged ? seg[s * span + k] : in[(size_t) (pl0 + s) * n + i]);
            acc[s].add(texel, w);
        }
    });
#pragma unroll
    for (int s = 0; s < K5_S; ++s)
        if (s < npl) out[(size_t) (pl0 + s) * n + x] = (uint16_t) unorm16(acc[s].result(sp));
}
// The same pass from the precomputed table (K5Table): no log / divide / sine per tap, the staged input converted to
// float once; per tap one coalesced 8-byte load, then per plane a shared-memory fetch, a multiply and the ordered add.
static_assert(K5_S == K5_S_PLANES && K5_XT == K5_BLOCK, "K5 table layout and kernel tile must agree");
template <bool AVG_ONLY, int S>
__global__ void __launch_bounds__(K5_BLOCK)
k5_table_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, int n, int count, const K5Table tb,
                const SmoothParams sp, int plane_stride, int plane_offset, int y0) {
    float* seg = reinterpret_cast<float*>(glb_smem);                  // [S][span] texels as float
    const int4 d = __ldg(tb.blk + blockIdx.x);
    const int base = d.x, taps = d.y, lo = d.z, span = d.w;
    const int pl0 = (y0 + (int) blockIdx.y) * S, npl = min(S, count - pl0);
    for (int i = threadIdx.x; i < S * span; i += K5_BLOCK) {
        const int pl = i / span, k = i - pl * span;
        seg[i] = pl < npl ? from16(in[((size_t) (pl0 + pl) * plane_stride + plane_offset) * n + lo + k]) : 0.0f;
    }
    __syncthreads();
    const int e = blockIdx.x * K5_BLOCK + threadIdx.x;               // output position
    if (e >= tb.count) return;
    const int x = tb.out ? __ldg(tb.out + e) : e;                     // texel it writes
    SmoothAcc acc[S];
#pragma unroll
    for (int s = 0; s < S; ++s) acc[s].init();
    const int2* col = tb.ent + base + threadIdx.x;
    for (int j = 0; j < taps; ++j) {
        const int2 t = __ldg(col + (size_t) j * K5_BLOCK);
        const float w = __int_as_float(t.y);
#pragma unroll
        for (int s = 0; s < S; ++s) {
            const float v = seg[s * span + t.x] * w;
            acc[s].avg += v;
            if (!AVG_ONLY) { if (acc[s].vmax < v) acc[s].vmax = v; }
        }
    }
    const float weight = __ldg(tb.wsum + e);
#pragma unroll
    for (int s = 0; s < S; ++s) {
        acc[s].weight = weight;
        if (s < npl) out[((size_t) (pl0 + s) * plane_stride + plane_offset) * n + x] = (uint16_t) unorm16(acc[s].result(sp));
    }
}

template <bool AVG_ONLY, int S>
static int launch_k5_table_t(const glava_b200_params& p, const uint16_t* d_in, uint16_t* d_out, int count, cudaStream_t st,
                             const K5Table& tb) {
    const SmoothParams sp = smooth_params(p);
    auto kern = k5_table_kernel<AVG_ONLY, S>;
    const int smem = S * tb.max_span * (int) sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "cudaFuncSetAttribute(k5 table): %s", cudaGetErrorString(e));
    }
    const unsigned gx = (tb.count + K5_BLOCK - 1) / K5_BLOCK;
    cudaError_t e = launch_y_slices((count + S - 1) / S, [&](int y0, unsigned rows) {
        kern<<<dim3(gx, rows), K5_BLOCK, smem, st>>>(d_in, d_out, p.n, count, tb, sp, 1, 0, y0);   // every plane in order
    });
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "smooth (table) kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

int launch_k5_full(const glava_b200_params& p, const SpectrumPlan& pl, const K5Table& table, const uint16_t* d_in,
                   uint16_t* d_out, int count, void* stream) {
    cudaStream_t st = (cudaStream_t) stream;
    if (pl.full_table) {
        // planes per CTA share every tap's index / weight load
        const bool avg = smooth_params(p).sample_mode == 0;
        switch (pl.table_planes) {
            case 8: return avg ? launch_k5_table_t<true, 8>(p, d_in, d_out, count, st, table)
                               : launch_k5_table_t<false, 8>(p, d_in, d_out, count, st, table);
            case 4: return avg ? launch_k5_table_t<true, 4>(p, d_in, d_out, count, st, table)
                               : launch_k5_table_t<false, 4>(p, d_in, d_out, count, st, table);
            default: return avg ? launch_k5_table_t<true, 2>(p, d_in, d_out, count, st, table)
                                : launch_k5_table_t<false, 2>(p, d_in, d_out, count, st, table);
        }
    }
    const size_t smem = k5_planes_smem(k5_planes_span(p));
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(k5_planes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
        if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "cudaFuncSetAttribute(k5): %s", cudaGetErrorString(e));
    }
    const unsigned gx = (p.n + K5_XT - 1) / K5_XT;
    cudaError_t e = launch_y_slices((count + K5_S - 1) / K5_S, [&](int y0, unsigned rows) {
        k5_planes_kernel<<<dim3(gx, rows), K5_XT, smem, st>>>(d_in, d_out, p.n, count, p, y0);
    });
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "smooth kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Need-list K5, lanes = streams.  Inside the spectrum kernel a texel's serial sum occupies one thread of a CTA whose other
// threads wait at a barrier.  Here one WARP owns one sampled
// texel of one channel for 32 * S streams: the tap list is the same for all of them, so a lane loads one {index, weight}
// of the next 32 taps (two coalesced loads) and the warp walks them by shuffle broadcast; per tap and stream one coalesced
// read of the transposed pre-smoothing texels (exported as float: converted once by the producer, not once per tap) and the
// ordered multiply-add of smooth_audio() (smooth.glsl:33-37).  S independent sums per lane share every broadcast.
// Pipeline B's state update (render.c:2177-2267: R16 upload, K1 max, K2 gravity, K3 ring, K4 average) as an elementwise
// kernel: one thread = 8 consecutive bins of one plane, every access a 16-byte vector (2 float4 of `spec`, one uint4 of each
// R16 plane), 2 + 1 + (F - 1) independent loads in flight per thread, full occupancy.  Inside the spectrum kernel the same
// work ran on the few warps of a plane's CTA behind the FFT's barriers: latency bound, 7x off the traffic it moves.
// Arithmetic = the in-kernel epilogue's (gravity_b, newest-first weighted average), bit for bit.
template <int FT>
__global__ void __launch_bounds__(128)
epilogue_b_kernel(const __grid_constant__ SpectrumArgs a, int n, int bins, int F, float diff, int y0, int rows) {
    // flat index over (plane of this slice, group of 8 bins): only the last CTA of a slice has idle threads
    const int groups = bins / 8, idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * groups) return;
    const int pr = idx / groups, plane = y0 + pr, n0 = (idx - pr * groups) * 8;
    const uint32_t um = a.umask ? __ldg(a.umask + (plane >> 1)) : 0x80000000u;
    if (!(um >> 31)) return;                                   // stream without new audio: state and texels stay
    const int out_idx = a.umask ? (int) (um & 0xffffu) : (int) (a.update % (unsigned long long) F);
    const size_t base = (size_t) plane * n + n0;
    const float4 s0 = *reinterpret_cast<const float4*>(a.spec + base), s1 = *reinterpret_cast<const float4*>(a.spec + base + 4);
    uint16_t* const grs = a.gr_store + base;
    uint16_t* const ring = a.ring_u + (size_t) plane * F * n + n0;
    const int FF = FT ? FT : F;
    uint4 gold = *reinterpret_cast<const uint4*>(grs);
    uint4 rg[FT ? FT : 1];
    if (FT > 1) {
#pragma unroll
        for (int i = 1; i < FT; ++i) { int fr = out_idx - i; if (fr < 0) fr += FT; rg[i] = *reinterpret_cast<const uint4*>(ring + (size_t) fr * n); }
    }
    const float v[8] = { s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w };
    const uint16_t* go = reinterpret_cast<const uint16_t*>(&gold);
    uint4 gnew, tex;
    uint16_t* gn = reinterpret_cast<uint16_t*>(&gnew); uint16_t* tx = reinterpret_cast<uint16_t*>(&tex);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const uint32_t gq = gravity_b(unorm16(v[e]), go[e], diff);
        gn[e] = (uint16_t) gq;
        uint32_t texel = gq;
        if (FF > 1) {
            float r = 0.0f;
            if (FT > 1) {
#pragma unroll
                for (int i = 0; i < FT; ++i) {                 // t0 = most recent (render.c:2250-2255)
                    const float t = from16(i == 0 ? gq : (uint32_t) reinterpret_cast<const uint16_t*>(&rg[i])[e]);
                    if (a.avg_b_windowed) r += a.avg_w_b[i] * t; else r += t;
                }
            } else {
                for (int i = 0; i < F; ++i) {
                    int fr = out_idx - i; if (fr < 0) fr += F;
                    const float t = from16(i == 0 ? gq : (uint32_t) ring[(size_t) fr * n + e]);
                    if (a.avg_b_windowed) r += a.avg_w_b[i] * t; else r += t;
                }
            }
            texel = unorm16(r / (float) FF);
        }
        tx[e] = (uint16_t) texel;
    }
    *reinterpret_cast<uint4*>(grs) = gnew;
    if (FF > 1) *reinterpret_cast<uint4*>(ring + (size_t) out_idx * n) = gnew;
    *reinterpret_cast<uint4*>(a.av_out + base) = tex;
}

// over the leading SpectrumPlan::epi_n bins of every plane (a multiple of 8)
static int launch_epilogue_b(const glava_b200_params& p, const SpectrumPlan& pl, const SpectrumArgs& a, cudaStream_t st) {
    const int planes = a.batch * 2, F = p.avg_frames, bins = pl.epi_n;
    const float diff = p.gravity_step * (1.0f / p.ur);
    // slices of at most GRID_Y_MAX planes keep the flat index in int (65535 planes x 2048 groups at 16384)
    cudaError_t e = launch_y_slices(planes, [&](int y0, unsigned rows) {
        const unsigned gx = (unsigned) (((long long) rows * (bins / 8) + 127) / 128);
#define GLB_EPI(FT) epilogue_b_kernel<FT><<<gx, 128, 0, st>>>(a, p.n, bins, F, diff, y0, (int) rows)
        switch (F) {
            case 5: GLB_EPI(5); break;                          // shipped default (smooth_parameters.glsl:56)
            case 6: GLB_EPI(6); break;                          // compiled-in default (render.c:912)
            case 3: GLB_EPI(3); break;
            case 4: GLB_EPI(4); break;
            default: GLB_EPI(0); break;
        }
#undef GLB_EPI
    });
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "epilogue kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

// [plane = stream * 2 + ch][bin] u16  ->  [ch][bin][stream] float (from16 applied once here, not once per tap): 32 x 32 tiles
// through shared memory, both sides coalesced.  A plane-owning spectrum CTA could only write its own stream's column of the
// transposed layout — 4-byte stores 4 KB apart — so the transposition is its own pass.
__global__ void __launch_bounds__(256)
av_transpose_kernel(const uint16_t* __restrict__ av, float* __restrict__ av_t, int n, int len, int batch) {
    __shared__ float tile[32][33];
    const int ch = blockIdx.z, b0 = blockIdx.x * 32, s0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;             // 32 x 8
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int s = s0 + ty + 8 * r, b = b0 + tx;
        tile[ty + 8 * r][tx] = (s < batch && b < len) ? from16(av[((size_t) s * 2 + ch) * n + b]) : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int b = b0 + ty + 8 * r, s = s0 + tx;
        if (b < len && s < batch) av_t[((size_t) ch * len + b) * batch + s] = tile[tx][ty + 8 * r];
    }
}

template <int MODE, int S, int D>
__global__ void __launch_bounds__(512)
k5_need_kernel(const float* __restrict__ av_t, int av_t_len, uint16_t* __restrict__ tex, int n, int batch, int channels,
               const unsigned char* __restrict__ csr, int csr_bytes, int csr_idx_off, int csr_off_off,
               const int* __restrict__ need, const float* __restrict__ wsum, int need_count, const SmoothParams sp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int groups = (batch + 32 * S - 1) / (32 * S);
    // consecutive warps take consecutive texels of the same stream group: their tap windows overlap, L1 serves the re-reads
    const int gw = blockIdx.x * (blockDim.x >> 5) + warp;
    // (the last texels of the list have the widest windows — scale_audio is log-like: they go first, the short ones fill the tail)
    const int k = need_count - 1 - gw % need_count, g = (gw / need_count) % groups, ch = gw / (need_count * groups);
    if (ch >= channels) return;
    const int x = __ldg(need + (size_t) ch * need_count + k);
    if (x < 0 || x >= n) return;
    const int stream0 = g * 32 * S + lane;
    const unsigned char* blob = csr + (size_t) ch * csr_bytes;
    const float*    tw = reinterpret_cast<const float*>(blob);
    const uint16_t* ti = reinterpret_cast<const uint16_t*>(blob + csr_idx_off);
    const int*      to = reinterpret_cast<const int*>(blob + csr_off_off);
    const int o0 = __ldg(to + k), o1 = __ldg(to + k + 1);
    // a lane past the batch reads column 0 (any valid address) and stores nothing
    const float* col[S];
#pragma unroll
    for (int q = 0; q < S; ++q) col[q] = av_t + (size_t) ch * av_t_len * batch + (stream0 + 32 * q < batch ? stream0 + 32 * q : 0);
    SmoothAcc acc[S];
#pragma unroll
    for (int q = 0; q < S; ++q) acc[q].init();
    for (int o = o0; o < o1; o += 32) {
        const int mine = o + lane;
        const int   my_i = mine < o1 ? (int) __ldg(ti + mine) * batch : 0;     // (a tap outside the texture is stored as index 0, weight 0)
        const float my_w = mine < o1 ? __ldg(tw + mine) : 0.0f;                 // (past the end of the list: index 0, weight 0 — adds +0)
        const int cnt = min(32, o1 - o);
        // groups of D taps: all D * S texel loads are issued before the first dependent add (the sums are serial, the
        // loads are not); a short last group runs past the list with weight 0 only when that cannot change a bit.
        // A warp's time is (taps / D) L2 round trips — the grid is about one wave of warps, so that chain IS the kernel's time
        for (int j0 = 0; j0 < cnt; j0 += D) {
            float t[D][S];
#pragma unroll
            for (int j = 0; j < D; ++j) {
                const int i = __shfl_sync(0xffffffffu, my_i, j0 + j);
#pragma unroll
                for (int q = 0; q < S; ++q) t[j][q] = __ldg(col[q] + i);
            }
            const int live = min(D, cnt - j0);
#pragma unroll
            for (int j = 0; j < D; ++j) {
                if (j < live) {                                            // (warp-uniform: the weight broadcast sits in the sum phase, D registers fewer)
                    const float wj = __shfl_sync(0xffffffffu, my_w, j0 + j);
#pragma unroll
                    for (int q = 0; q < S; ++q) { if (MODE == 0) acc[q].avg += t[j][q] * wj; else acc[q].add_noweight(t[j][q], wj); }
                }
            }
        }
    }
    const float weight = __ldg(wsum + (size_t) ch * need_count + k);
#pragma unroll
    for (int q = 0; q < S; ++q) {
        acc[q].weight = weight;
        const int stream = stream0 + 32 * q;
        if (stream < batch) tex[((size_t) stream * 2 + ch) * n + x] = (uint16_t) unorm16(acc[q].result(sp));
    }
}

// The same sums out of shared memory.  A CTA = (channel, 32 streams, block of sampled texels whose tap windows overlap:
// tables.h build_need_blocks): the union of the block's windows is staged once, straight from the [plane][bin] R16 texture —
// a warp reads a stream's bins with coalesced 32-bit loads, converts (from16, once per staged texel) and stores them
// TRANSPOSED, tile[bin][stream] with a row stride of 33 floats, so that the tap loop's reads (lanes = streams) and these
// writes (lanes = bins) are both conflict-free to 2-way.  No transposed copy in HBM, no av_transpose_kernel, and the tap
// loop's traffic leaves L2: k5_need_kernel moves 4 bytes per tap and lane through L2, its bound.
template <int MODE>
__global__ void __launch_bounds__(512)
k5_need_smem_kernel(const uint16_t* __restrict__ av, uint16_t* __restrict__ tex, int n, int batch,
                    const unsigned char* __restrict__ csr, int csr_bytes, int csr_idx_off, int csr_off_off,
                    const int* __restrict__ need, const float* __restrict__ wsum, int need_count,
                    const int4* __restrict__ blocks, int nblk, const SmoothParams sp) {
    extern __shared__ float k5n_tile[];                                  // [rows][33]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int ch = blockIdx.z, g = blockIdx.y;
    const int4 bk = __ldg(blocks + (size_t) ch * nblk + (nblk - 1 - blockIdx.x));      // the widest windows (last texels) first
    const int k0 = bk.x, k1 = bk.y, lo = bk.z, rows = bk.w;
    if (k1 <= k0) return;
    for (int s = warp; s < 32; s += nwarps) {
        const int stream = g * 32 + s;
        if (stream < batch) {
            const uint32_t* src = reinterpret_cast<const uint32_t*>(av + ((size_t) stream * 2 + ch) * n + lo);   // n, lo even: 4-byte aligned
            for (int c = lane; c < (rows >> 1); c += 32) {
                const uint32_t u = __ldg(src + c);
                k5n_tile[(2 * c) * 33 + s] = from16(u & 0xffffu);
                k5n_tile[(2 * c + 1) * 33 + s] = from16(u >> 16);
            }
        } else {
            for (int c = lane; c < rows; c += 32) k5n_tile[c * 33 + s] = 0.0f;      // lanes past the batch sum zeros and store nothing
        }
    }
    __syncthreads();
    const unsigned char* blob = csr + (size_t) ch * csr_bytes;
    const float*    tw = reinterpret_cast<const float*>(blob);
    const uint16_t* ti = reinterpret_cast<const uint16_t*>(blob + csr_idx_off);
    const int*      to = reinterpret_cast<const int*>(blob + csr_off_off);
    const int stream = g * 32 + lane;
    const float* col = k5n_tile + lane;
    for (int k = k1 - 1 - warp; k >= k0; k -= nwarps) {
        const int x = __ldg(need + (size_t) ch * need_count + k);
        if (x < 0 || x >= n) continue;
        const int o0 = __ldg(to + k), o1 = __ldg(to + k + 1);
        SmoothAcc acc; acc.init();
        for (int o = o0; o < o1; o += 32) {
            const int mine = o + lane;
            // (a tap outside the texture is stored as index 0, weight 0: any row of the tile times +0 adds the same +0)
            int my_r = 0; float my_w = 0.0f;
            if (mine < o1) { my_r = (int) __ldg(ti + mine) - lo; my_r = my_r < 0 ? 0 : (my_r >= rows ? rows - 1 : my_r); my_r *= 33; my_w = __ldg(tw + mine); }
            const int cnt = min(32, o1 - o);
#pragma unroll 8
            for (int j = 0; j < cnt; ++j) {
                const int r = __shfl_sync(0xffffffffu, my_r, j);
                const float w = __shfl_sync(0xffffffffu, my_w, j);
                const float t = col[r];
                if (MODE == 0) acc.avg += t * w; else acc.add_noweight(t, w);
            }
        }
        acc.weight = __ldg(wsum + (size_t) ch * need_count + k);
        if (stream < batch) tex[((size_t) stream * 2 + ch) * n + x] = (uint16_t) unorm16(acc.result(sp));
    }
}

// the need-list K5 kernels read the pre-smoothing texture a.av_out and write the sampled texels of a.tex
static int launch_k5_need_smem(const glava_b200_params& p, const SpectrumPlan& pl, const SpectrumDevTables& tb,
                               const SpectrumArgs& a, cudaStream_t st) {
    const SmoothParams sp = smooth_params(p);
    if (tb.need_nblk <= 0) return 0;
    const size_t smem = (size_t) tb.need_max_rows * 33 * sizeof(float);
    const int channels = p.module != GLAVA_B200_MOD_WAVE ? 2 : 1;
    dim3 grid((unsigned) tb.need_nblk, (unsigned) ((a.batch + 31) / 32), (unsigned) channels);
    auto kern = sp.sample_mode == 0 ? k5_need_smem_kernel<0> : k5_need_smem_kernel<1>;
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem)) != cudaSuccess)
        return fail(GLAVA_B200_ECUDA, "need-list smooth kernel shared memory %zu: %s", smem, cudaGetErrorString(e));
    kern<<<grid, pl.k5n_warps * 32, smem, st>>>(a.av_out, a.tex, p.n, a.batch, tb.csr, tb.csr_bytes, tb.csr_idx_off, tb.csr_off_off,
                                                tb.need, tb.tap_wsum, tb.need_count, reinterpret_cast<const int4*>(tb.need_blk),
                                                tb.need_nblk, sp);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail(GLAVA_B200_ECUDA, "need-list smooth kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

static int launch_k5_need(const glava_b200_params& p, const SpectrumPlan& pl, const SpectrumDevTables& tb, const SpectrumArgs& a,
                          cudaStream_t st) {
    const SmoothParams sp = smooth_params(p);
    const int batch = a.batch, channels = p.module != GLAVA_B200_MOD_WAVE ? 2 : 1, av_t_len = pl.av_t_len;
    {
        dim3 tg((av_t_len + 31) / 32, (batch + 31) / 32, channels);
        av_transpose_kernel<<<tg, 256, 0, st>>>(a.av_out, tb.av_t, p.n, av_t_len, batch);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "transpose kernel launch: %s", cudaGetErrorString(e));
    }
    // S streams per lane share every tap broadcast (spectrum_plan.h chooses S from the batch)
    const int S = pl.k5n_s, wpc = pl.k5n_warps;
    const int groups = (batch + 32 * S - 1) / (32 * S);
    const long long warps = (long long) channels * tb.need_count * groups;
    // warps per CTA = consecutive texels of one stream group: their tap windows overlap almost entirely, so the more of them
    // share an SM's L1 the fewer reads go to L2 (the kernel moves 4 bytes per tap and lane: L2 bandwidth is its bound)
    const unsigned grid = (unsigned) ((warps + wpc - 1) / wpc);
    if (grid == 0) return 0;
#define GLB_K5N(M, SS, DD) k5_need_kernel<M, SS, DD><<<grid, wpc * 32, 0, st>>>(tb.av_t, av_t_len, a.tex, p.n, batch, channels, tb.csr, \
                                                 tb.csr_bytes, tb.csr_idx_off, tb.csr_off_off, tb.need, tb.tap_wsum, tb.need_count, sp)
#define GLB_K5N_M(SS, DD) do { if (sp.sample_mode == 0) GLB_K5N(0, SS, DD); else GLB_K5N(1, SS, DD); } while (0)
    if (S == 4) GLB_K5N_M(4, 8);
    else if (S == 2) GLB_K5N_M(2, 8);
    else GLB_K5N_M(1, 8);
#undef GLB_K5N_M
#undef GLB_K5N
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "need-list smooth kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

int launch_spectrum_update(const glava_b200_params& p, const SpectrumPlan& pl, const SpectrumDevTables& tb, const SpectrumArgs& in,
                           void* stream) {
    cudaStream_t st = (cudaStream_t) stream;
    const bool need_in_kernel = pl.k5 == K5Form::TAPS_SMEM || pl.k5 == K5Form::TAPS_L2 || pl.k5 == K5Form::TAPS_DIRECT;
    const bool need_kernel = pl.k5 == K5Form::NEED_SMEM || pl.k5 == K5Form::NEED_L2;
    // full-plane smoothing (every texel wanted): the spectrum kernel exports the pre-smoothing texture and a second kernel
    // smooths all planes, sharing the tap weights between planes
    const bool full_kernel = !in.skip_tex && (pl.k5 == K5Form::FULL_TABLE || pl.k5 == K5Form::FULL_PLANES);
    SpectrumArgs a = in;
    a.need = need_in_kernel ? tb.need : nullptr; a.need_count = tb.need_count;
    a.tap_tab = need_in_kernel ? tb.tap_tab : nullptr; a.tap_cnt = tb.tap_cnt; a.tap_wsum = tb.tap_wsum; a.tap_max = tb.tap_max;
    a.tap_ku = pl.tap_ku;
    a.epi_n = pl.epi_n;
    a.csr = pl.k5 == K5Form::TAPS_SMEM ? tb.csr : nullptr; a.csr_bytes = tb.csr_bytes; a.csr_idx_off = tb.csr_idx_off; a.csr_off_off = tb.csr_off_off;
    a.variant_oop = pl.fft_oop; a.variant_t = pl.fft_t;
    a.av_out = (full_kernel || need_kernel) ? in.av_out : nullptr;
    a.av_t_len = need_kernel ? pl.av_t_len : 0;
    // three-kernel form of the lazy pipeline-B update: transform_fft only in the plane-per-CTA kernel, the R16 state update as
    // an elementwise kernel, K5 on (texel, stream) pairs.  Every F: at F = 1 epilogue_b_kernel<0> keeps no ring.
    a.fft_only = pl.split_epilogue ? 1 : 0;
    int rc;
    if ((rc = launch_spectrum(p, pl, a, st)) != 0) return rc;
    if (pl.split_epilogue && (rc = launch_epilogue_b(p, pl, a, st)) != 0) return rc;
    if (pl.k5 == K5Form::NEED_SMEM && (rc = launch_k5_need_smem(p, pl, tb, a, st)) != 0) return rc;
    if (pl.k5 == K5Form::NEED_L2 && (rc = launch_k5_need(p, pl, tb, a, st)) != 0) return rc;
    // wave uses plane 0 of each stream only; smoothing the (zero) odd planes too keeps the launch simple
    if (full_kernel && (rc = launch_k5_full(p, pl, tb.k5, a.av_out, a.tex, a.batch * 2, stream)) != 0) return rc;
    // NEED_L2: av_transpose_kernel + k5_need_kernel
    return 1 + pl.split_epilogue + (pl.k5 == K5Form::NEED_SMEM) + 2 * (pl.k5 == K5Form::NEED_L2) + full_kernel;
}

// ---------------------------------------------------------------------------------------------
// FIFO ingest (fifo.c:89-110): slide + append, ping-pong between two ring buffers
// FLOAT_IN: the samples are already float (PulseAudio backend, pulse_input.c:146-174: stored as they are, the mono mix is
// (l + r) / 2 in float); otherwise int16 (fifo.c: s16 / 65535.f, integer mean for mono)
template <bool FLOAT_IN>
__global__ void fifo_ingest_kernel(const void* __restrict__ chunks, int frames, int n, int channels,
                                   const float* __restrict__ src_l, const float* __restrict__ src_r,
                                   float* __restrict__ dst_l, float* __restrict__ dst_r, int y0) {
    const int s = y0 + (int) blockIdx.y;
    const size_t base = (size_t) s * n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float l, r;
        if (i < n - frames) { l = src_l[base + i + frames]; r = src_r[base + i + frames]; }
        else {
            const int q = i - (n - frames);
            if (FLOAT_IN) {
                const float* in = reinterpret_cast<const float*>(chunks) + (size_t) s * frames * 2;
                const float a = in[2 * q], b = in[2 * q + 1];
                if (channels == 1) { const float m = (a + b) / 2; l = m; r = m; }
                else { l = a; r = b; }
            } else {
                const int16_t* in = reinterpret_cast<const int16_t*>(chunks) + (size_t) s * frames * 2;
                const int a = in[2 * q], b = in[2 * q + 1];
                if (channels == 1) { float m = (float) ((a + b) / 2) / (float) 65535; l = m; r = m; }
                else { l = (float) a / (float) 65535; r = (float) b / (float) 65535; }
            }
        }
        dst_l[base + i] = l; dst_r[base + i] = r;
    }
}
int launch_fifo_ingest(const glava_b200_params& p, const void* d_chunks, bool float_in, int frames, const float* src_l, const float* src_r,
                       float* dst_l, float* dst_r, int batch, void* stream) {
    const unsigned gx = (p.n + 1023) / 1024;
    const int chans = (p.mirror_input || p.channels == 1) ? 1 : 2;       // the AUDIO side's mono mix (setmirror), not the shader's _CHANNELS
    cudaStream_t st = (cudaStream_t) stream;
    cudaError_t e = launch_y_slices(batch, [&](int y0, unsigned rows) {
        if (float_in) fifo_ingest_kernel<true><<<dim3(gx, rows), 256, 0, st>>>(d_chunks, frames, p.n, chans, src_l, src_r, dst_l, dst_r, y0);
        else fifo_ingest_kernel<false><<<dim3(gx, rows), 256, 0, st>>>(d_chunks, frames, p.n, chans, src_l, src_r, dst_l, dst_r, y0);
    });
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "fifo ingest kernel launch: %s", cudaGetErrorString(e));
    return 0;
}

}  // namespace glb
