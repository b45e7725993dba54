// export_kernels.cu — glava_b200_export_frames (DESIGN 4.10): the current frames of a list of streams, flipped
// top-down and written as RGBA / BGRA (optionally composited) or NV12 into the caller's device buffers.
//
// One launch per call.  The list (destination, framebuffer slot) reaches the device in one small copy; the grid is
// flattened over (listed entry, output row pair, 128-pixel strip) on grid.x only, one warp per item, so any list length
// and frame size fit.  A thread owns a quad of pixels on both rows of its pair: two 16-byte loads, then two 16-byte
// streaming stores (RGBA / BGRA) or two 4-byte Y stores and one 4-byte CbCr store (NV12).  With dirty-row marks the warp
// reads only the rows its strip's band words say may be non-zero (export_core.h); every other row is zero pixels that are
// never loaded.  Widths that are not a multiple of 4 take a per-pixel tail.
//
// glava_b200_export_scaled (DESIGN 4.11) is export_scaled_kernel below: the same frames, cropped and shrunk by the exact
// area average of export_core.h, in one launch with its own argument struct.  glava_b200_overlay_frames (DESIGN 4.12) is
// overlay_kernel: the same frames composited onto the caller's images in place, likewise with its own argument struct.
// Both take entries with a chroma pointer (ExportEntryUV); export_kernel keeps ExportEntry.  glava_b200_export_ladder
// (DESIGN 4.13) is export_ladder_kernel: every rung of every entry in one launch, each unit run by the per-item body of
// the rung's standalone kernel.  I420, YUV 4:4:4 and P010 (DESIGN 4.14) run kernels of their own with the same items
// (export_yuv_kernel, export_scaled_yuv_kernel, export_ladder_yuv_kernel), as do the planar 10-bit formats (DESIGN 4.16:
// export_p10_kernel, export_scaled_p10_kernel, export_ladder_p10_kernel) and the 4:2:2 formats (DESIGN 4.18:
// export_422_kernel, export_scaled_422_kernel, export_ladder_422_kernel).  The host half is export.cpp.
#include "internal.h"
#include "export_core.h"

#include <cuda_runtime.h>

#include <type_traits>

namespace glb {

static_assert(sizeof(LadderRung) == 80, "LadderRung keeps its size: enc sits in what was padding");
static_assert(sizeof(LadderArgs{}.yuv[0]) == 24, "LadderArgs keeps its size: za sits in what was padding");
static_assert(sizeof(OverlayArgs) == 72 && sizeof(OverlayPlanesArgs) == 80, "the overlay arguments keep their size: fade sits in "
              "what was padding");

// f(std::integral_constant<int, E>()) for the encoding E = enc, 1..3 (DESIGN 4.15): the launchers run these instantiations
// for any encoding but 0, whose kernels are the ones every call without a colour bit ran before there were encodings
template <typename F>
static void for_enc(int enc, F&& f) {
    if (enc == 1) f(std::integral_constant<int, 1>());
    else if (enc == 2) f(std::integral_constant<int, 2>());
    else f(std::integral_constant<int, 3>());
}

// whether row y of the strip must be read (false: it is all zero in memory)
template <typename A>
__device__ __forceinline__ bool row_read(const A& a, int slot, int y, int strip) {
    if (!a.marks) return true;
    return export_row_read(__ldg(a.marks + export_mark_index(slot, a.w, a.h, a.mark_rows, y, strip)), y);
}

// Framebuffer loads.  A standalone export reads each line once, so it streams them (evict-first, ld.global.cs); the ladder
// reads a line once per rung and wants the later rungs to find it in L2, so it loads at normal priority (Keep: ld.global.cg)
template <bool Keep>
__device__ __forceinline__ uint4 fb_load4(const uint32_t* p) {
    return Keep ? __ldcg(reinterpret_cast<const uint4*>(p)) : __ldcs(reinterpret_cast<const uint4*>(p));
}
template <bool Keep>
__device__ __forceinline__ uint32_t fb_load(const uint32_t* p) { return Keep ? __ldcg(p) : __ldcs(p); }

// the quad at x of framebuffer row y of a w-pixel-wide frame (pixels past the right edge read as 0)
template <bool Keep = false>
__device__ __forceinline__ void load_quad(const uint32_t* frame, int w, int y, int x, uint32_t px[4]) {
    const uint32_t* row = frame + (size_t) y * w;
    if ((w & 3) == 0) {                                     // rows are 16-byte aligned
        const uint4 v = fb_load4<Keep>(row + x);
        px[0] = v.x; px[1] = v.y; px[2] = v.z; px[3] = v.w;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) px[k] = x + k < w ? fb_load<Keep>(row + x + k) : 0u;
    }
}

// The grid of one launch over `items` warp items, 8 per CTA: grid-stride beyond 16 CTAs per SM of an H100 SXM, with 32-bit
// item arithmetic whenever the item count allows (every realistic list: 1024 1080p frames are 8.3 M row-pair items)
struct ExportGrid { unsigned blocks; bool narrow; };
static ExportGrid export_grid(uint64_t items) {
    const uint64_t blocks = (items + 7) / 8;
    const unsigned grid = blocks < 132u * 16u ? (unsigned) (blocks ? blocks : 1) : 132u * 16u;
    return { grid, items + ((uint64_t) grid << 3) < (1ull << 32) };
}

static int launch_status(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GLAVA_B200_ECUDA, "%s kernel launch: %s", what, cudaGetErrorString(e));
    return 0;
}

// zpx: what a zero pixel becomes (a quad of zero pixels skips the per-pixel arithmetic)
__device__ __forceinline__ void store_rgba(const ExportFmt& f, uint8_t* row, int x, int w, const uint32_t in[4], uint32_t zpx) {
    uint32_t px[4] = { zpx, zpx, zpx, zpx };
    if ((in[0] | in[1] | in[2] | in[3]) != 0u) {
#pragma unroll
        for (int k = 0; k < 4; ++k) px[k] = export_px(f, in[k]);
    }
    uint32_t* out = reinterpret_cast<uint32_t*>(row) + x;
    if (x + 4 <= w) __stcs(reinterpret_cast<uint4*>(out), make_uint4(px[0], px[1], px[2], px[3]));   // pitch and dst: multiples of 16
    else
        for (int k = 0; k < 4 && x + k < w; ++k) __stcs(out + k, px[k]);
}

// One item of export_kernel (and of a ladder's whole-frame rung): output rows 2j and 2j + 1 (framebuffer rows h - 1 - 2j and
// h - 2 - 2j) of the quad at x of `strip`; the NV12 CbCr plane's row 0 is dst + uv_offset; zy / zuv / zpx: what zero pixels
// become.  E: the encoding of NV12 (DESIGN 4.15).
// A reads w, h, marks, mark_rows, format and pitch.
template <bool Keep, int E = 0, typename A>
__device__ __forceinline__ void export_item(const A& a, const ExportFmt& f, const uint32_t* frame, int slot, uint8_t* dst,
                                            size_t uv_offset, int j, int strip, int x, uint32_t zy, uint32_t zuv, uint32_t zpx) {
    const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
    if (row_read(a, slot, y0, strip)) load_quad<Keep>(frame, a.w, y0, x, top);
    if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad<Keep>(frame, a.w, y1, x, bot);
    uint8_t* const r0 = dst + (size_t) (2 * j) * a.pitch;
    if (a.format == GLAVA_B200_EXPORT_NV12) {               // h even: both rows exist
        uint32_t yt = zy, yb = zy, c = zuv;
        if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) != 0u) c = export_nv12_quad<E>(f, top, bot, &yt, &yb);
        uint8_t* const pu = dst + uv_offset + (size_t) j * a.pitch + x;
        if (x + 4 <= a.w) {
            __stcs(reinterpret_cast<uint32_t*>(r0 + x), yt);
            __stcs(reinterpret_cast<uint32_t*>(r0 + a.pitch + x), yb);
            __stcs(reinterpret_cast<uint32_t*>(pu), c);
        } else {                                            // w even: the last two pixels of a row
            __stcs(reinterpret_cast<unsigned short*>(r0 + x), (unsigned short) yt);
            __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch + x), (unsigned short) yb);
            __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) c);
        }
    } else {
        store_rgba(f, r0, x, a.w, top, zpx);
        if (y1 >= 0) store_rgba(f, r0 + a.pitch, x, a.w, bot, zpx);
    }
}

template <typename Index>
__global__ void __launch_bounds__(256) export_kernel(const __grid_constant__ ExportArgs a) {
    const ExportFmt f = { a.format, a.over, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    // what zero pixels become: most of a frame is zero rows the marks skip, and most of the rest is zero pixels
    const uint32_t zero4[4] = { 0u, 0u, 0u, 0u };
    uint32_t zy, zy1;
    const uint32_t zuv = export_nv12_quad(f, zero4, zero4, &zy, &zy1), zpx = export_px(f, 0u);
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        // export_item<false>(a, ..., a.uv_offset, ...) written out: called, ptxas orders four register moves of zpx
        // differently, and this kernel keeps the machine code it was measured with
        const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
        uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
        if (row_read(a, slot, y0, strip)) load_quad(frame, a.w, y0, x, top);
        if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad(frame, a.w, y1, x, bot);
        uint8_t* const r0 = dst + (size_t) (2 * j) * a.pitch;
        if (a.format == GLAVA_B200_EXPORT_NV12) {           // h even: both rows exist
            uint32_t yt = zy, yb = zy, uv = zuv;
            if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) != 0u) uv = export_nv12_quad(f, top, bot, &yt, &yb);
            uint8_t* const pu = dst + a.uv_offset + (size_t) j * a.pitch + x;
            if (x + 4 <= a.w) {
                __stcs(reinterpret_cast<uint32_t*>(r0 + x), yt);
                __stcs(reinterpret_cast<uint32_t*>(r0 + a.pitch + x), yb);
                __stcs(reinterpret_cast<uint32_t*>(pu), uv);
            } else {                                        // w even: the last two pixels of a row
                __stcs(reinterpret_cast<unsigned short*>(r0 + x), (unsigned short) yt);
                __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch + x), (unsigned short) yb);
                __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) uv);
            }
        } else {
            store_rgba(f, r0, x, a.w, top, zpx);
            if (y1 >= 0) store_rgba(f, r0 + a.pitch, x, a.w, bot, zpx);
        }
    }
}

// export_kernel's NV12 under encoding E = 1..3 (DESIGN 4.15): the same items, run by export_item
template <typename Index, int E>
__global__ void __launch_bounds__(256) export_nv12_enc_kernel(const __grid_constant__ ExportArgs a) {
    const ExportFmt f = { GLAVA_B200_EXPORT_NV12, 1, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const uint32_t zero4[4] = { 0u, 0u, 0u, 0u };
    uint32_t zy, zy1;
    const uint32_t zuv = export_nv12_quad<E>(f, zero4, zero4, &zy, &zy1);
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        export_item<false, E>(a, f, frame, slot, dst, a.uv_offset, j, strip, x, zy, zuv, 0u);
    }
}

// ---- I420, YUV 4:4:4 and P010 (DESIGN 4.14) --------------------------------------------------------------------------------
// export_kernel's items (output row pair x 128-pixel strip, a quad per lane) with the new formats' stores, in kernels of their
// own so that export_kernel keeps its machine code.  I420: two 4-byte Y stores and a 2-byte Cb and a 2-byte Cr store
// (chroma rows pitch / 2 apart); YUV 4:4:4: a 4-byte Y, Cb and Cr store per row; P010: an 8-byte Y store per row and an
// 8-byte CbCr store.  Past the last full quad: I420 and P010 have an even width (the last two pixels of a row), YUV 4:4:4
// stores byte by byte.

// the first n (1..4) bytes of v at p (n == 4: p is 4-byte aligned)
__device__ __forceinline__ void store_bytes(uint8_t* p, uint32_t v, int n) {
    if (n >= 4) __stcs(reinterpret_cast<uint32_t*>(p), v);
    else
        for (int k = 0; k < n; ++k) __stcs(p + k, (uint8_t) (v >> (8 * k)));
}

// YUV 4:4:4 of one row's quad: n pixels of Y at py, Cb at pu and Cr cr bytes past it
template <int E>
__device__ __forceinline__ void store_444(const ExportFmt& f, const uint32_t q[4], uint8_t* py, uint8_t* pu, size_t cr, int n,
                                          const ExportZero& z) {
    uint32_t y = z.y, u = z.u, v = z.v;
    if ((q[0] | q[1] | q[2] | q[3]) != 0u) export_444_quad<E>(f, q, &y, &u, &v);
    store_bytes(py, y, n);
    store_bytes(pu, u, n);
    store_bytes(pu + cr, v, n);
}

// One item of export_yuv_kernel (and of a ladder's whole-frame I420 / YUV444 / P010 rung): as export_item, with the chroma
// plane at `cb` (I420 / YUV444: Cb, Cr `cr` bytes further; P010: CbCr) and z what zero pixels become.  fmt: a constant in
// the standalone kernels, the rung's format in the ladder; E the encoding.  A reads w, h, marks, mark_rows and pitch.
template <bool Keep, int E = 0, typename A>
__device__ __forceinline__ void yuv_item(const A& a, const ExportFmt& f, int fmt, const uint32_t* frame, int slot, uint8_t* dst,
                                         uint8_t* cb, size_t cr, int j, int strip, int x, const ExportZero& z) {
    const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
    if (row_read(a, slot, y0, strip)) load_quad<Keep>(frame, a.w, y0, x, top);
    if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad<Keep>(frame, a.w, y1, x, bot);
    uint8_t* const r0 = dst + (size_t) (2 * j) * a.pitch;
    const bool full = x + 4 <= a.w;
    if (fmt == GLAVA_B200_EXPORT_YUV444) {                  // any w and h
        const int n = full ? 4 : a.w - x;
        const size_t o = (size_t) (2 * j) * a.pitch + x;
        store_444<E>(f, top, dst + o, cb + o, cr, n, z);
        if (y1 >= 0) store_444<E>(f, bot, dst + o + a.pitch, cb + o + a.pitch, cr, n, z);
        return;
    }
    const bool any = (top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) != 0u;
    if (fmt == GLAVA_B200_EXPORT_I420) {                    // w and h even
        uint32_t yt = z.y, yb = z.y, u = z.u, v = z.v;
        if (any) {
            const uint32_t uv = export_nv12_quad<E>(f, top, bot, &yt, &yb);
            u = export_cb_pair(uv); v = export_cr_pair(uv);
        }
        uint8_t* const pu = cb + (size_t) j * (a.pitch >> 1) + (x >> 1);
        if (full) {
            __stcs(reinterpret_cast<uint32_t*>(r0 + x), yt);
            __stcs(reinterpret_cast<uint32_t*>(r0 + a.pitch + x), yb);
            __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
            __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) v);
        } else {                                            // the last two pixels of a row
            __stcs(reinterpret_cast<unsigned short*>(r0 + x), (unsigned short) yt);
            __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch + x), (unsigned short) yb);
            __stcs(pu, (uint8_t) u);
            __stcs(pu + cr, (uint8_t) v);
        }
        return;
    }
    uint32_t yt[2] = { z.y, z.y }, yb[2] = { z.y, z.y }, uv[2] = { z.u, z.u };   // P010, w and h even
    if (any) export_p010_quad<E>(f, top, bot, yt, yb, uv);
    uint8_t* const pu = cb + (size_t) j * a.pitch + 2 * x;
    if (full) {
        __stcs(reinterpret_cast<uint2*>(r0 + 2 * x), make_uint2(yt[0], yt[1]));
        __stcs(reinterpret_cast<uint2*>(r0 + a.pitch + 2 * x), make_uint2(yb[0], yb[1]));
        __stcs(reinterpret_cast<uint2*>(pu), make_uint2(uv[0], uv[1]));
    } else {
        __stcs(reinterpret_cast<uint32_t*>(r0 + 2 * x), yt[0]);
        __stcs(reinterpret_cast<uint32_t*>(r0 + a.pitch + 2 * x), yb[0]);
        __stcs(reinterpret_cast<uint32_t*>(pu), uv[0]);
    }
}

template <typename Index, int Fmt, int E>
__device__ __forceinline__ void yuv_loop(const ExportArgs& a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const ExportZero z = export_zero<E>(f);                 // once per thread, as export_kernel's constants
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        yuv_item<false, E>(a, f, Fmt, frame, slot, dst, dst + a.uv_offset, a.cr_offset, j, strip, x, z);
    }
}

template <typename Index, int Fmt>
__global__ void __launch_bounds__(256) export_yuv_kernel(const __grid_constant__ ExportArgs a) { yuv_loop<Index, Fmt, 0>(a); }
// under encoding E = 1..3
template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_yuv_enc_kernel(const __grid_constant__ ExportArgs a) { yuv_loop<Index, Fmt, E>(a); }

template <typename Index>
static void launch_yuv(const ExportArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.enc) {
        for_enc(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (a.format == GLAVA_B200_EXPORT_I420) export_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_I420, E><<<blocks, 256, 0, st>>>(a);
            else if (a.format == GLAVA_B200_EXPORT_YUV444) export_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_YUV444, E><<<blocks, 256, 0, st>>>(a);
            else export_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_P010, E><<<blocks, 256, 0, st>>>(a);
        });
    } else if (a.format == GLAVA_B200_EXPORT_I420) export_yuv_kernel<Index, GLAVA_B200_EXPORT_I420><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV444) export_yuv_kernel<Index, GLAVA_B200_EXPORT_YUV444><<<blocks, 256, 0, st>>>(a);
    else export_yuv_kernel<Index, GLAVA_B200_EXPORT_P010><<<blocks, 256, 0, st>>>(a);
}

// ---- planar 10-bit: YUV420P10 and YUV444P10 (DESIGN 4.16) -----------------------------------------------------------------
// export_kernel's items again, with little-endian uint16 samples holding the 10-bit code in their low bits: YUV420P10 an
// 8-byte Y store per row and a 4-byte Cb and a 4-byte Cr store (chroma rows pitch / 2 apart), YUV444P10 an 8-byte Y, Cb and
// Cr store per row.  Past the last full quad YUV420P10 has an even width (the last two pixels of a row) and YUV444P10
// stores sample by sample.  These kernels have no earlier form to keep, so all four encodings are instantiations of one
// template.

// f(std::integral_constant<int, E>()) for the encoding E = enc, 0..3
template <typename F>
static void for_any_enc(int enc, F&& f) {
    if (enc == 0) f(std::integral_constant<int, 0>());
    else for_enc(enc, f);
}

// f(std::integral_constant<int, E>()) for the HDR encoding E = enc, 4 (PQ) or 5 (HLG) (DESIGN 4.22): the launchers route
// these to new instantiations of the 10-bit kernels before for_enc / for_any_enc, so no existing kernel sees them
template <typename F>
static void for_hdr(int enc, F&& f) {
    if (enc == GLB_ENC_PQ) f(std::integral_constant<int, GLB_ENC_PQ>());
    else f(std::integral_constant<int, GLB_ENC_HLG>());
}

// the first n (1..4) uint16 samples of the words v[0], v[1] at p (n == 4: p is 8-byte aligned); the tail is written out,
// since indexing v by a run-time sample number puts the words on the stack
__device__ __forceinline__ void store_u16(uint8_t* p, const uint32_t v[2], int n) {
    unsigned short* const q = reinterpret_cast<unsigned short*>(p);
    if (n >= 4) {
        __stcs(reinterpret_cast<uint2*>(p), make_uint2(v[0], v[1]));
        return;
    }
    __stcs(q, (unsigned short) v[0]);
    if (n > 1) __stcs(q + 1, (unsigned short) (v[0] >> 16));
    if (n > 2) __stcs(q + 2, (unsigned short) v[1]);
}

// YUV444P10 of one row's quad: n samples of Y at py, Cb at pu and Cr cr bytes past it
template <int E>
__device__ __forceinline__ void store_444p10(const ExportFmt& f, const uint32_t q[4], uint8_t* py, uint8_t* pu, size_t cr, int n,
                                             const ExportZero& z) {
    uint32_t y[2] = { z.y, z.y }, u[2] = { z.u, z.u }, v[2] = { z.v, z.v };
    if ((q[0] | q[1] | q[2] | q[3]) != 0u) export_444p10_quad<E>(f, q, y, u, v);
    store_u16(py, y, n);
    store_u16(pu, u, n);
    store_u16(pu + cr, v, n);
}

// One item of export_p10_kernel (and of a ladder's whole-frame planar 10-bit rung), as yuv_item: the Cb plane at `cb`, Cr
// `cr` bytes further; z what zero pixels become (export_zero10).  A reads w, h, marks, mark_rows and pitch.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void p10_item(const A& a, const ExportFmt& f, int fmt, const uint32_t* frame, int slot, uint8_t* dst,
                                         uint8_t* cb, size_t cr, int j, int strip, int x, const ExportZero& z) {
    const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
    if (row_read(a, slot, y0, strip)) load_quad<Keep>(frame, a.w, y0, x, top);
    if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad<Keep>(frame, a.w, y1, x, bot);
    const size_t o = (size_t) (2 * j) * a.pitch + 2 * (size_t) x;
    const bool full = x + 4 <= a.w;
    if (fmt == GLAVA_B200_EXPORT_YUV444P10) {               // any w and h
        const int n = full ? 4 : a.w - x;
        store_444p10<E>(f, top, dst + o, cb + o, cr, n, z);
        if (y1 >= 0) store_444p10<E>(f, bot, dst + o + a.pitch, cb + o + a.pitch, cr, n, z);
        return;
    }
    uint32_t yt[2] = { z.y, z.y }, yb[2] = { z.y, z.y }, u = z.u, v = z.v;   // YUV420P10, w and h even
    if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) != 0u) export_i010_quad<E>(f, top, bot, yt, yb, &u, &v);
    uint8_t* const pu = cb + (size_t) j * (a.pitch >> 1) + x;   // x / 2 samples of 2 bytes
    if (full) {
        __stcs(reinterpret_cast<uint2*>(dst + o), make_uint2(yt[0], yt[1]));
        __stcs(reinterpret_cast<uint2*>(dst + o + a.pitch), make_uint2(yb[0], yb[1]));
        __stcs(reinterpret_cast<uint32_t*>(pu), u);
        __stcs(reinterpret_cast<uint32_t*>(pu + cr), v);
    } else {                                                // the last two pixels of a row
        __stcs(reinterpret_cast<uint32_t*>(dst + o), yt[0]);
        __stcs(reinterpret_cast<uint32_t*>(dst + o + a.pitch), yb[0]);
        __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
        __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) v);
    }
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_p10_kernel(const __grid_constant__ ExportArgs a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const ExportZero z = export_zero10<E>(f);               // once per thread, as export_kernel's constants
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        p10_item<false, E>(a, f, Fmt, frame, slot, dst, dst + a.uv_offset, a.cr_offset, j, strip, x, z);
    }
}

template <typename Index>
static void launch_p10(const ExportArgs& a, unsigned blocks, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUV420P10) export_p10_kernel<Index, GLAVA_B200_EXPORT_YUV420P10, E><<<blocks, 256, 0, st>>>(a);
        else export_p10_kernel<Index, GLAVA_B200_EXPORT_YUV444P10, E><<<blocks, 256, 0, st>>>(a);
    });
}

// ---- 4:2:2: YUV422P, YUV422P10 and UYVY (DESIGN 4.18) ----------------------------------------------------------------------
// export_kernel's items once more (output row pair x 128-pixel strip, a quad per lane), each row converted on its own, so an
// odd h leaves the last pair one row.  Per lane per row: YUV422P a 4-byte Y store and a 2-byte Cb and a 2-byte Cr store
// (chroma rows pitch / 2 apart), YUV422P10 an 8-byte Y store and a 4-byte Cb and a 4-byte Cr store, UYVY one 8-byte store.
// Past the last full quad the width is 4k + 2: the last pixel pair of a row.  All four encodings are instantiations of one
// template, as the planar 10-bit kernels are.

// One row of a 4:2:2 item: the quad q at x of output row r (dst: row 0's luma or UYVY bytes, cb: row 0's Cb, Cr `cr` bytes
// further); full: a whole quad, else the last pixel pair; z what zero pixels become (export_zero422)
template <int E>
__device__ __forceinline__ void row_422(const ExportFmt& f, int fmt, const uint32_t q[4], uint8_t* dst, uint8_t* cb, size_t cr,
                                        size_t pitch, int r, int x, bool full, const ExportZero& z) {
    const bool any = (q[0] | q[1] | q[2] | q[3]) != 0u;
    if (fmt == GLAVA_B200_EXPORT_UYVY) {
        uint32_t w[2] = { z.y, z.y };
        if (any) {
            uint32_t y;
            const uint32_t uv = export_422_quad<E>(f, q, &y);
            export_uyvy_words(y, uv, w);
        }
        uint8_t* const p = dst + (size_t) r * pitch + 2 * (size_t) x;
        if (full) __stcs(reinterpret_cast<uint2*>(p), make_uint2(w[0], w[1]));
        else __stcs(reinterpret_cast<uint32_t*>(p), w[0]);
    } else if (fmt == GLAVA_B200_EXPORT_YUV422P) {
        uint32_t y = z.y, u = z.u, v = z.v;
        if (any) {
            const uint32_t uv = export_422_quad<E>(f, q, &y);
            u = export_cb_pair(uv); v = export_cr_pair(uv);
        }
        uint8_t* const py = dst + (size_t) r * pitch + x;
        uint8_t* const pu = cb + (size_t) r * (pitch >> 1) + (x >> 1);
        if (full) {
            __stcs(reinterpret_cast<uint32_t*>(py), y);
            __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
            __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) v);
        } else {
            __stcs(reinterpret_cast<unsigned short*>(py), (unsigned short) y);
            __stcs(pu, (uint8_t) u);
            __stcs(pu + cr, (uint8_t) v);
        }
    } else {                                                // YUV422P10
        uint32_t y[2] = { z.y, z.y }, u = z.u, v = z.v;
        if (any) export_422p10_quad<E>(f, q, y, &u, &v);
        uint8_t* const py = dst + (size_t) r * pitch + 2 * (size_t) x;
        uint8_t* const pu = cb + (size_t) r * (pitch >> 1) + x;   // x / 2 samples of 2 bytes
        if (full) {
            __stcs(reinterpret_cast<uint2*>(py), make_uint2(y[0], y[1]));
            __stcs(reinterpret_cast<uint32_t*>(pu), u);
            __stcs(reinterpret_cast<uint32_t*>(pu + cr), v);
        } else {
            __stcs(reinterpret_cast<uint32_t*>(py), y[0]);
            __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
            __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) v);
        }
    }
}

// One item of export_422_kernel (and of a ladder's whole-frame 4:2:2 rung), as p10_item.  A reads w, h, marks, mark_rows
// and pitch.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void item_422(const A& a, const ExportFmt& f, int fmt, const uint32_t* frame, int slot, uint8_t* dst,
                                         uint8_t* cb, size_t cr, int j, int strip, int x, const ExportZero& z) {
    const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
    if (row_read(a, slot, y0, strip)) load_quad<Keep>(frame, a.w, y0, x, top);
    if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad<Keep>(frame, a.w, y1, x, bot);
    const bool full = x + 4 <= a.w;
    row_422<E>(f, fmt, top, dst, cb, cr, a.pitch, 2 * j, x, full, z);
    if (y1 >= 0) row_422<E>(f, fmt, bot, dst, cb, cr, a.pitch, 2 * j + 1, x, full, z);
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_422_kernel(const __grid_constant__ ExportArgs a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const ExportZero z = export_zero422<E>(f);              // once per thread, as export_kernel's constants
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        item_422<false, E>(a, f, Fmt, frame, slot, dst, dst + a.uv_offset, a.cr_offset, j, strip, x, z);
    }
}

template <typename Index>
static void launch_422(const ExportArgs& a, unsigned blocks, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUV422P) export_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P, E><<<blocks, 256, 0, st>>>(a);
        else if (a.format == GLAVA_B200_EXPORT_YUV422P10) export_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P10, E><<<blocks, 256, 0, st>>>(a);
        else export_422_kernel<Index, GLAVA_B200_EXPORT_UYVY, E><<<blocks, 256, 0, st>>>(a);
    });
}

// ---- transparency: YUVA420P, YUVA444P10 and straight RGBA / BGRA (DESIGN 4.19) ---------------------------------------------
// export_kernel's items once more (output row pair x 128-pixel strip, a quad per lane).  Per lane: YUVA420P two 4-byte Y
// stores, a 2-byte Cb and a 2-byte Cr store and two 4-byte A stores (A rows pitch apart, one Cb to Cr distance past Cr);
// YUVA444P10 an 8-byte Y, Cb, Cr and A store per row; straight RGBA / BGRA a 16-byte store per row.  Past the last full quad
// YUVA420P has an even width (the last two pixels of a row), the others store pixel by pixel.  Straight RGBA / BGRA run
// under their kernel format code (export_core.h GLB_EXPORT_STRAIGHT) and encoding 0 only.

// YUVA444P10 of one row's quad: n samples of Y at py, Cb at pu, Cr cr and A 2 cr bytes past it
template <int E>
__device__ __forceinline__ void store_yuva444p10(const ExportFmt& f, const uint32_t q[4], uint8_t* py, uint8_t* pu, size_t cr, int n,
                                                 const ExportZeroA& z) {
    uint32_t y[2] = { z.y, z.y }, u[2] = { z.u, z.u }, v[2] = { z.v, z.v }, al[2] = { z.a, z.a };
    if ((q[0] | q[1] | q[2] | q[3]) != 0u) export_yuva444p10_quad<E>(f, q, y, u, v, al);
    store_u16(py, y, n);
    store_u16(pu, u, n);
    store_u16(pu + cr, v, n);
    store_u16(pu + 2 * cr, al, n);
}

// straight RGBA / BGRA of one row's quad at x (fmt: the kernel format code; zpx what a zero pixel becomes)
__device__ __forceinline__ void store_straight(const ExportFmt& f, int fmt, uint8_t* row, int x, int w, const uint32_t in[4],
                                               uint32_t zpx) {
    uint32_t px[4] = { zpx, zpx, zpx, zpx };
    if ((in[0] | in[1] | in[2] | in[3]) != 0u) {
#pragma unroll
        for (int k = 0; k < 4; ++k) px[k] = export_straight_out(f, fmt, in[k]);
    }
    uint32_t* out = reinterpret_cast<uint32_t*>(row) + x;
    if (x + 4 <= w) __stcs(reinterpret_cast<uint4*>(out), make_uint4(px[0], px[1], px[2], px[3]));
    else
        for (int k = 0; k < 4 && x + k < w; ++k) __stcs(out + k, px[k]);
}

// One item of export_yuva_kernel (and of a ladder's whole-frame alpha rung), as p10_item: the Cb plane at `cb`, Cr `cr`
// bytes further, A `cr` bytes past Cr; z what zero pixels become (export_zero_alpha).  A reads w, h, marks, mark_rows and
// pitch.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void yuva_item(const A& a, const ExportFmt& f, int fmt, const uint32_t* frame, int slot, uint8_t* dst,
                                          uint8_t* cb, size_t cr, int j, int strip, int x, const ExportZeroA& z) {
    const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
    uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
    if (row_read(a, slot, y0, strip)) load_quad<Keep>(frame, a.w, y0, x, top);
    if (y1 >= 0 && row_read(a, slot, y1, strip)) load_quad<Keep>(frame, a.w, y1, x, bot);
    const bool full = x + 4 <= a.w;
    if (export_straight(fmt)) {                             // any w and h
        uint8_t* const r0 = dst + (size_t) (2 * j) * a.pitch;
        store_straight(f, fmt, r0, x, a.w, top, z.y);
        if (y1 >= 0) store_straight(f, fmt, r0 + a.pitch, x, a.w, bot, z.y);
        return;
    }
    if (fmt == GLAVA_B200_EXPORT_YUVA444P10) {              // any w and h
        const int n = full ? 4 : a.w - x;
        const size_t o = (size_t) (2 * j) * a.pitch + 2 * (size_t) x;
        store_yuva444p10<E>(f, top, dst + o, cb + o, cr, n, z);
        if (y1 >= 0) store_yuva444p10<E>(f, bot, dst + o + a.pitch, cb + o + a.pitch, cr, n, z);
        return;
    }
    uint32_t yt = z.y, yb = z.y, u = z.u, v = z.v, at = z.a, ab = z.a;   // YUVA420P, w and h even
    if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) != 0u)
        export_yuva420_quad<E>(f, top, bot, &yt, &yb, &u, &v, &at, &ab);
    const size_t o = (size_t) (2 * j) * a.pitch + x;
    uint8_t* const pu = cb + (size_t) j * (a.pitch >> 1) + (x >> 1);
    uint8_t* const pa = cb + 2 * cr + o;
    if (full) {
        __stcs(reinterpret_cast<uint32_t*>(dst + o), yt);
        __stcs(reinterpret_cast<uint32_t*>(dst + o + a.pitch), yb);
        __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
        __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) v);
        __stcs(reinterpret_cast<uint32_t*>(pa), at);
        __stcs(reinterpret_cast<uint32_t*>(pa + a.pitch), ab);
    } else {                                                // the last two pixels of a row
        __stcs(reinterpret_cast<unsigned short*>(dst + o), (unsigned short) yt);
        __stcs(reinterpret_cast<unsigned short*>(dst + o + a.pitch), (unsigned short) yb);
        __stcs(pu, (uint8_t) u);
        __stcs(pu + cr, (uint8_t) v);
        __stcs(reinterpret_cast<unsigned short*>(pa), (unsigned short) at);
        __stcs(reinterpret_cast<unsigned short*>(pa + a.pitch), (unsigned short) ab);
    }
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_yuva_kernel(const __grid_constant__ ExportArgs a) {
    const ExportFmt f = { Fmt, a.over, a.native, a.bg };
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + 1) >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    const ExportZeroA z = export_zero_alpha<E>(f);          // once per thread, as export_kernel's constants
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int j = (int) (rem / strips), strip = (int) (rem - (Index) j * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntry* e = a.list + k;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        yuva_item<false, E>(a, f, Fmt, frame, slot, dst, dst + a.uv_offset, a.cr_offset, j, strip, x, z);
    }
}

template <typename Index>
static void launch_yuva(const ExportArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.format == (GLAVA_B200_EXPORT_RGBA | GLB_EXPORT_STRAIGHT))
        export_yuva_kernel<Index, GLAVA_B200_EXPORT_RGBA | GLB_EXPORT_STRAIGHT, 0><<<blocks, 256, 0, st>>>(a);
    else if (a.format == (GLAVA_B200_EXPORT_BGRA | GLB_EXPORT_STRAIGHT))
        export_yuva_kernel<Index, GLAVA_B200_EXPORT_BGRA | GLB_EXPORT_STRAIGHT, 0><<<blocks, 256, 0, st>>>(a);
    else for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUVA420P) export_yuva_kernel<Index, GLAVA_B200_EXPORT_YUVA420P, E><<<blocks, 256, 0, st>>>(a);
        else export_yuva_kernel<Index, GLAVA_B200_EXPORT_YUVA444P10, E><<<blocks, 256, 0, st>>>(a);
    });
}

// ---- BT.2020 HDR (DESIGN 4.22): P010, YUV420P10, YUV444P10 and YUV422P10 under E = 4 / 5 -------------------------------
// The 10-bit kernels' own items, instantiated for the HDR encodings (export_core.h's quads branch on E at compile time)
template <typename Index, int E>
static void launch_hdr(const ExportArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.format == GLAVA_B200_EXPORT_P010) export_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_P010, E><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV420P10) export_p10_kernel<Index, GLAVA_B200_EXPORT_YUV420P10, E><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV444P10) export_p10_kernel<Index, GLAVA_B200_EXPORT_YUV444P10, E><<<blocks, 256, 0, st>>>(a);
    else export_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P10, E><<<blocks, 256, 0, st>>>(a);
}

int launch_export(const ExportArgs& a, void* stream) {
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) ((a.w + 127) >> 7) * (uint64_t) ((a.h + 1) >> 1));
    cudaStream_t st = (cudaStream_t) stream;
    if (a.enc >= GLB_ENC_PQ) {
        for_hdr(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (g.narrow) launch_hdr<uint32_t, E>(a, g.blocks, st);
            else launch_hdr<uint64_t, E>(a, g.blocks, st);
        });
        return launch_status("export");
    }
    if (export_alpha(a.format)) {
        if (g.narrow) launch_yuva<uint32_t>(a, g.blocks, st);
        else launch_yuva<uint64_t>(a, g.blocks, st);
    } else if (export_422(a.format)) {
        if (g.narrow) launch_422<uint32_t>(a, g.blocks, st);
        else launch_422<uint64_t>(a, g.blocks, st);
    } else if (export_p10(a.format)) {
        if (g.narrow) launch_p10<uint32_t>(a, g.blocks, st);
        else launch_p10<uint64_t>(a, g.blocks, st);
    } else if (a.enc && a.format == GLAVA_B200_EXPORT_NV12) {
        for_enc(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (g.narrow) export_nv12_enc_kernel<uint32_t, E><<<g.blocks, 256, 0, st>>>(a);
            else export_nv12_enc_kernel<uint64_t, E><<<g.blocks, 256, 0, st>>>(a);
        });
    } else if (a.format != GLAVA_B200_EXPORT_NV12 && export_yuv(a.format)) {
        if (g.narrow) launch_yuv<uint32_t>(a, g.blocks, (cudaStream_t) stream);
        else launch_yuv<uint64_t>(a, g.blocks, (cudaStream_t) stream);
    } else if (g.narrow) export_kernel<uint32_t><<<g.blocks, 256, 0, (cudaStream_t) stream>>>(a);
    else export_kernel<uint64_t><<<g.blocks, 256, 0, (cudaStream_t) stream>>>(a);
    return launch_status("export");
}

// ---- glava_b200_export_scaled (DESIGN 4.11) --------------------------------------------------------------------------------
// The grid is flattened over (listed entry, output row — NV12: row pair —, run of 32 output columns) on grid.x, one warp per
// item, lane = output column.  With marks a lane walks its footprint strip by strip and, within a strip, band by band of the dirty-row
// marks (export_band_rows): one mark word per band says which of its rows may be non-zero, and only those rows are visited,
// so the rows of a band the marks call empty cost one load together (visiting every footprint row and loading its word
// made the headline thumbnails slower than the full-size export).  A visited row's span is summed from aligned quads
// (16-byte loads when rows are 16-byte aligned; neighbouring lanes read neighbouring segments) in 32-bit per channel and
// folded into 64-bit sums with the row's weight.  NV12 chroma takes the right neighbour's pixels of both rows by shuffle.

// output pixel (X, Y) of the lane, before any R / B swap; active = false: a lane past out_w (the sums stay empty).  A reads
// w, h, marks, mark_rows and the rectangle (src_*, out_*) as ScaledArgs names them.
template <bool Keep, typename A>
__device__ __forceinline__ uint32_t scaled_px(const A& a, const ExportFmt& f, const uint32_t* frame, int slot, int Y,
                                              bool active, const ExportSpan& sx, const ExportRecip& rcp, uint32_t zc) {
    const ExportSpan sy = export_span(Y, a.src_h, a.out_h);
    const int x0 = a.src_x + sx.first, x1 = a.src_x + sx.last;
    // framebuffer rows [yb, ye) of the footprint; row y is crop row h - 1 - src_y - y
    const int yb = export_fb_row(a.h, a.src_y, sy.last), ye = export_fb_row(a.h, a.src_y, sy.first) + 1;
    const int rows = a.marks ? a.mark_rows : 0;
    uint64_t acc[4] = { 0u, 0u, 0u, 0u }, wsum = 0u;
    // without marks the whole span is one pass (strip by strip, a lane whose span straddles strips would hold its warp)
    for (int strip = x0 >> 7, last = rows ? x1 >> 7 : strip; active && strip <= last; ++strip) {
        const int qa = max(x0, strip << 7) & ~3, qb = rows ? min(x1, (strip << 7) + 127) : x1;
        for (int y = yb; y < ye;) {
            int ra, rb;
            const uint32_t mark = rows ? __ldg(a.marks + export_mark_index(slot, a.w, a.h, rows, y, strip)) : 0u;
            y = export_band_rows(y, ye, rows, mark, &ra, &rb);
            for (int yy = ra; yy < rb; ++yy) {
                const uint32_t* src = frame + (size_t) yy * a.w;
                uint32_t row[4] = { 0u, 0u, 0u, 0u }, row_w = 0u;
                for (int qx = qa; qx <= qb; qx += 4) {
                    uint32_t px[4];
                    if ((a.w & 3) == 0) {
                        const uint4 v = fb_load4<Keep>(src + qx);
                        px[0] = v.x; px[1] = v.y; px[2] = v.z; px[3] = v.w;
                    } else {
#pragma unroll
                        for (int k = 0; k < 4; ++k) px[k] = qx + k >= x0 && qx + k <= x1 ? fb_load<Keep>(src + qx + k) : 0u;
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int x = qx + k;
                        if (x >= x0 && x <= x1) export_acc(f, px[k], export_span_weight(sx, x - a.src_x, a.out_w), row, &row_w);
                    }
                }
                export_fold(row, row_w, export_span_weight(sy, a.h - 1 - a.src_y - yy, a.out_h), acc, &wsum);
            }
        }
    }
    return export_scaled_px(f, acc, wsum, (uint64_t) a.src_w * (uint64_t) a.src_h, rcp, zc);
}

// One item of export_scaled_kernel (and of a ladder's other rungs): output row u (NV12: rows 2u and 2u + 1) at column X of
// the lane; zc: what a zero pixel becomes; E the encoding of NV12.  A as scaled_px, and fb, format and pitch.
template <bool Keep, int E = 0, typename A>
__device__ __forceinline__ void scaled_item(const A& a, const ExportFmt& f, const ExportRecip& rcp, uint32_t zc, bool nv12,
                                            const ExportEntryUV* e, int u, int X, int lane) {
    const bool active = X < a.out_w;
    const int slot = __ldg(&e->slot);
    const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
    const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
    uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    if (nv12) {                                             // out_w even: the whole 2x2 block is in this warp
        const uint32_t top = scaled_px<Keep>(a, f, frame, slot, 2 * u, active, sx, rcp, zc);
        const uint32_t bot = scaled_px<Keep>(a, f, frame, slot, 2 * u + 1, active, sx, rcp, zc);
        const uint32_t top1 = __shfl_down_sync(0xffffffffu, top, 1), bot1 = __shfl_down_sync(0xffffffffu, bot, 1);
        if (!active) return;
        uint8_t* const r0 = dst + (size_t) (2 * u) * a.pitch + X;
        __stcs(r0, (uint8_t) export_y<E>(top));
        __stcs(r0 + a.pitch, (uint8_t) export_y<E>(bot));
        if (!(lane & 1)) {
            uint8_t* const uv = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
            __stcs(reinterpret_cast<unsigned short*>(uv + (size_t) u * a.pitch + X),
                   (unsigned short) export_cbcr<E>(export_avg4(top, top1, bot, bot1)));
        }
    } else {
        uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
        if (!active) return;
        if (a.format == GLAVA_B200_EXPORT_BGRA) px = export_swap_rb(px);
        __stcs(reinterpret_cast<uint32_t*>(dst + (size_t) u * a.pitch) + X, px);
    }
}

template <typename Index, int E>
__device__ __forceinline__ void scaled_loop(const ScaledArgs& a) {
    const ExportFmt f = { a.format, a.over, a.native, a.bg };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const bool nv12 = a.format == GLAVA_B200_EXPORT_NV12;
    const uint32_t zc = f.over ? export_over(0u, f.bg, f.native) : 0u;   // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) (nv12 ? a.out_h >> 1 : a.out_h);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        scaled_item<false, E>(a, f, rcp, zc, nv12, a.list + k, u, X, lane);
    }
}

template <typename Index>
__global__ void __launch_bounds__(256) export_scaled_kernel(const __grid_constant__ ScaledArgs a) { scaled_loop<Index, 0>(a); }
// NV12 under encoding E = 1..3
template <typename Index, int E>
__global__ void __launch_bounds__(256) export_scaled_enc_kernel(const __grid_constant__ ScaledArgs a) { scaled_loop<Index, E>(a); }

// One item of export_scaled_yuv_kernel (and of a ladder's other I420 / YUV444 / P010 rungs), as scaled_item: output row u
// (I420 / P010: rows 2u and 2u + 1, the chroma of each 2x2 block from the right neighbour by shuffle) at column X of the
// lane.  The chroma plane is the entry's dst_uv (I420 / YUV444: Cb, Cr `cr` bytes further; P010: CbCr); E the encoding.
template <bool Keep, int E = 0, typename A>
__device__ __forceinline__ void scaled_yuv_item(const A& a, const ExportFmt& f, int fmt, const ExportRecip& rcp, uint32_t zc,
                                                size_t cr, const ExportEntryUV* e, int u, int X, int lane) {
    const bool active = X < a.out_w;
    const int slot = __ldg(&e->slot);
    const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
    const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
    uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
    if (fmt == GLAVA_B200_EXPORT_YUV444) {
        const uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
        if (!active) return;
        const size_t o = (size_t) u * a.pitch + X;
        const uint32_t uv = export_cbcr<E>(px);
        __stcs(dst + o, (uint8_t) export_y<E>(px));
        __stcs(cb + o, (uint8_t) uv);
        __stcs(cb + cr + o, (uint8_t) (uv >> 8));
        return;
    }
    // out_w even: the whole 2x2 block is in this warp
    const uint32_t top = scaled_px<Keep>(a, f, frame, slot, 2 * u, active, sx, rcp, zc);
    const uint32_t bot = scaled_px<Keep>(a, f, frame, slot, 2 * u + 1, active, sx, rcp, zc);
    const uint32_t top1 = __shfl_down_sync(0xffffffffu, top, 1), bot1 = __shfl_down_sync(0xffffffffu, bot, 1);
    if (!active) return;
    if (fmt == GLAVA_B200_EXPORT_I420) {
        uint8_t* const r0 = dst + (size_t) (2 * u) * a.pitch + X;
        __stcs(r0, (uint8_t) export_y<E>(top));
        __stcs(r0 + a.pitch, (uint8_t) export_y<E>(bot));
        if (!(lane & 1)) {
            const uint32_t uv = export_cbcr<E>(export_avg4(top, top1, bot, bot1));
            uint8_t* const pu = cb + (size_t) u * (a.pitch >> 1) + (X >> 1);
            __stcs(pu, (uint8_t) uv);
            __stcs(pu + cr, (uint8_t) (uv >> 8));
        }
    } else {                                                // P010
        uint8_t* const r0 = dst + (size_t) (2 * u) * a.pitch + 2 * X;
        __stcs(reinterpret_cast<unsigned short*>(r0), (unsigned short) (export_y10<E>(top) << 6));
        __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch), (unsigned short) (export_y10<E>(bot) << 6));
        if (!(lane & 1))
            __stcs(reinterpret_cast<uint32_t*>(cb + (size_t) u * a.pitch + 2 * X), export_block10<E>(top, top1, bot, bot1) << 6);
    }
}

template <typename Index, int Fmt, int E>
__device__ __forceinline__ void scaled_yuv_loop(const ScaledArgs& a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const uint32_t zc = export_over(0u, f.bg, f.native);    // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) (Fmt == GLAVA_B200_EXPORT_YUV444 ? a.out_h : a.out_h >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        scaled_yuv_item<false, E>(a, f, Fmt, rcp, zc, a.cr_offset, a.list + k, u, X, lane);
    }
}

template <typename Index, int Fmt>
__global__ void __launch_bounds__(256) export_scaled_yuv_kernel(const __grid_constant__ ScaledArgs a) { scaled_yuv_loop<Index, Fmt, 0>(a); }
// under encoding E = 1..3
template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_scaled_yuv_enc_kernel(const __grid_constant__ ScaledArgs a) {
    scaled_yuv_loop<Index, Fmt, E>(a);
}

template <typename Index>
static void launch_scaled_yuv(const ScaledArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.enc) {
        for_enc(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (a.format == GLAVA_B200_EXPORT_I420) export_scaled_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_I420, E><<<blocks, 256, 0, st>>>(a);
            else if (a.format == GLAVA_B200_EXPORT_YUV444) export_scaled_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_YUV444, E><<<blocks, 256, 0, st>>>(a);
            else export_scaled_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_P010, E><<<blocks, 256, 0, st>>>(a);
        });
    } else if (a.format == GLAVA_B200_EXPORT_I420) export_scaled_yuv_kernel<Index, GLAVA_B200_EXPORT_I420><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV444) export_scaled_yuv_kernel<Index, GLAVA_B200_EXPORT_YUV444><<<blocks, 256, 0, st>>>(a);
    else export_scaled_yuv_kernel<Index, GLAVA_B200_EXPORT_P010><<<blocks, 256, 0, st>>>(a);
}

// One item of export_scaled_p10_kernel (and of a ladder's other planar 10-bit rungs), as scaled_yuv_item: output row u
// (YUV420P10: rows 2u and 2u + 1, the chroma of each 2x2 block from the right neighbour by shuffle) at column X of the lane,
// one uint16 sample per store.  The Cb plane is the entry's dst_uv, Cr `cr` bytes further; E the encoding.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void scaled_p10_item(const A& a, const ExportFmt& f, int fmt, const ExportRecip& rcp, uint32_t zc,
                                                size_t cr, const ExportEntryUV* e, int u, int X, int lane) {
    const bool active = X < a.out_w;
    const int slot = __ldg(&e->slot);
    const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
    const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
    uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
    if (fmt == GLAVA_B200_EXPORT_YUV444P10) {
        const uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
        if (!active) return;
        const size_t o = (size_t) u * a.pitch + 2 * (size_t) X;
        const uint32_t uv = export_cbcr10_px<E>(px);
        __stcs(reinterpret_cast<unsigned short*>(dst + o), (unsigned short) export_y10<E>(px));
        __stcs(reinterpret_cast<unsigned short*>(cb + o), (unsigned short) uv);
        __stcs(reinterpret_cast<unsigned short*>(cb + cr + o), (unsigned short) (uv >> 16));
        return;
    }
    // YUV420P10, out_w even: the whole 2x2 block is in this warp
    const uint32_t top = scaled_px<Keep>(a, f, frame, slot, 2 * u, active, sx, rcp, zc);
    const uint32_t bot = scaled_px<Keep>(a, f, frame, slot, 2 * u + 1, active, sx, rcp, zc);
    const uint32_t top1 = __shfl_down_sync(0xffffffffu, top, 1), bot1 = __shfl_down_sync(0xffffffffu, bot, 1);
    if (!active) return;
    uint8_t* const r0 = dst + (size_t) (2 * u) * a.pitch + 2 * (size_t) X;
    __stcs(reinterpret_cast<unsigned short*>(r0), (unsigned short) export_y10<E>(top));
    __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch), (unsigned short) export_y10<E>(bot));
    if (!(lane & 1)) {
        const uint32_t uv = export_block10<E>(top, top1, bot, bot1);
        uint8_t* const pu = cb + (size_t) u * (a.pitch >> 1) + X;   // X / 2 samples of 2 bytes
        __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) uv);
        __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) (uv >> 16));
    }
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_scaled_p10_kernel(const __grid_constant__ ScaledArgs a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const uint32_t zc = export_over(0u, f.bg, f.native);    // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) (Fmt == GLAVA_B200_EXPORT_YUV444P10 ? a.out_h : a.out_h >> 1);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        scaled_p10_item<false, E>(a, f, Fmt, rcp, zc, a.cr_offset, a.list + k, u, X, lane);
    }
}

template <typename Index>
static void launch_scaled_p10(const ScaledArgs& a, unsigned blocks, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUV420P10) export_scaled_p10_kernel<Index, GLAVA_B200_EXPORT_YUV420P10, E><<<blocks, 256, 0, st>>>(a);
        else export_scaled_p10_kernel<Index, GLAVA_B200_EXPORT_YUV444P10, E><<<blocks, 256, 0, st>>>(a);
    });
}

// One item of export_scaled_422_kernel (and of a ladder's other 4:2:2 rungs), as scaled_p10_item: output row u at column X
// of the lane (out_w even: a pixel pair is an even lane and its right neighbour, whose pixel comes by shuffle).  The even
// lane of a pair stores its chroma (UYVY: the pair's whole word).  The Cb plane is the entry's dst_uv, Cr `cr` bytes
// further; E the encoding.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void scaled_422_item(const A& a, const ExportFmt& f, int fmt, const ExportRecip& rcp, uint32_t zc,
                                                size_t cr, const ExportEntryUV* e, int u, int X, int lane) {
    const bool active = X < a.out_w;
    const int slot = __ldg(&e->slot);
    const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
    const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
    uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    const uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
    const uint32_t px1 = __shfl_down_sync(0xffffffffu, px, 1);
    if (!active) return;
    if (fmt == GLAVA_B200_EXPORT_UYVY) {
        if (!(lane & 1)) {
            const uint32_t uv = export_cbcr<E>(export_avg4(px, px1, px, px1));
            __stcs(reinterpret_cast<uint32_t*>(dst + (size_t) u * a.pitch + 2 * (size_t) X),
                   (uv & 0xffu) | (export_y<E>(px) << 8) | ((uv & 0xff00u) << 8) | (export_y<E>(px1) << 24));
        }
        return;
    }
    uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
    if (fmt == GLAVA_B200_EXPORT_YUV422P) {
        __stcs(dst + (size_t) u * a.pitch + X, (uint8_t) export_y<E>(px));
        if (!(lane & 1)) {
            const uint32_t uv = export_cbcr<E>(export_avg4(px, px1, px, px1));
            uint8_t* const pu = cb + (size_t) u * (a.pitch >> 1) + (X >> 1);
            __stcs(pu, (uint8_t) uv);
            __stcs(pu + cr, (uint8_t) (uv >> 8));
        }
    } else {                                                // YUV422P10
        __stcs(reinterpret_cast<unsigned short*>(dst + (size_t) u * a.pitch + 2 * (size_t) X), (unsigned short) export_y10<E>(px));
        if (!(lane & 1)) {
            const uint32_t uv = export_block10<E>(px, px1, px, px1);
            uint8_t* const pu = cb + (size_t) u * (a.pitch >> 1) + X;   // X / 2 samples of 2 bytes
            __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) uv);
            __stcs(reinterpret_cast<unsigned short*>(pu + cr), (unsigned short) (uv >> 16));
        }
    }
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_scaled_422_kernel(const __grid_constant__ ScaledArgs a) {
    const ExportFmt f = { Fmt, 1, a.native, a.bg };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const uint32_t zc = export_over(0u, f.bg, f.native);    // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) a.out_h;
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        scaled_422_item<false, E>(a, f, Fmt, rcp, zc, a.cr_offset, a.list + k, u, X, lane);
    }
}

template <typename Index>
static void launch_scaled_422(const ScaledArgs& a, unsigned blocks, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUV422P) export_scaled_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P, E><<<blocks, 256, 0, st>>>(a);
        else if (a.format == GLAVA_B200_EXPORT_YUV422P10) export_scaled_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P10, E><<<blocks, 256, 0, st>>>(a);
        else export_scaled_422_kernel<Index, GLAVA_B200_EXPORT_UYVY, E><<<blocks, 256, 0, st>>>(a);
    });
}

// One item of export_scaled_yuva_kernel (and of a ladder's other alpha rungs), as scaled_p10_item: output row u (YUVA420P:
// rows 2u and 2u + 1, the chroma of each 2x2 block from the right neighbour by shuffle) at column X of the lane.  scaled_px
// with f.over unset averages the stored channels, alpha included (export_scaled RGBA without EXPORT_OVER); the alpha
// arithmetic then runs on that premultiplied image.  The Cb plane is the entry's dst_uv, Cr `cr` bytes further, A `cr`
// bytes past Cr; fmt the kernel format code, E the encoding.
template <bool Keep, int E, typename A>
__device__ __forceinline__ void scaled_yuva_item(const A& a, const ExportFmt& f, int fmt, const ExportRecip& rcp, uint32_t zc,
                                                 size_t cr, const ExportEntryUV* e, int u, int X, int lane) {
    const bool active = X < a.out_w;
    const int slot = __ldg(&e->slot);
    const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
    const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
    uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    if (export_straight(fmt)) {
        const uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
        if (!active) return;
        const uint32_t s = export_straight_px(px);
        __stcs(reinterpret_cast<uint32_t*>(dst + (size_t) u * a.pitch) + X,
               (fmt & ~GLB_EXPORT_STRAIGHT) == GLAVA_B200_EXPORT_BGRA ? export_swap_rb(s) : s);
        return;
    }
    uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
    if (fmt == GLAVA_B200_EXPORT_YUVA444P10) {
        const uint32_t px = scaled_px<Keep>(a, f, frame, slot, u, active, sx, rcp, zc);
        if (!active) return;
        const uint32_t s = export_straight_px(px), uv = export_cbcr10_px<E>(s);
        const size_t o = (size_t) u * a.pitch + 2 * (size_t) X;
        __stcs(reinterpret_cast<unsigned short*>(dst + o), (unsigned short) export_y10<E>(s));
        __stcs(reinterpret_cast<unsigned short*>(cb + o), (unsigned short) uv);
        __stcs(reinterpret_cast<unsigned short*>(cb + cr + o), (unsigned short) (uv >> 16));
        __stcs(reinterpret_cast<unsigned short*>(cb + 2 * cr + o), (unsigned short) export_a10(px >> 24));
        return;
    }
    // YUVA420P, out_w even: the whole 2x2 block is in this warp
    const uint32_t top = scaled_px<Keep>(a, f, frame, slot, 2 * u, active, sx, rcp, zc);
    const uint32_t bot = scaled_px<Keep>(a, f, frame, slot, 2 * u + 1, active, sx, rcp, zc);
    const uint32_t top1 = __shfl_down_sync(0xffffffffu, top, 1), bot1 = __shfl_down_sync(0xffffffffu, bot, 1);
    if (!active) return;
    const size_t o = (size_t) (2 * u) * a.pitch + X;
    __stcs(dst + o, (uint8_t) export_y<E>(export_straight_px(top)));
    __stcs(dst + o + a.pitch, (uint8_t) export_y<E>(export_straight_px(bot)));
    __stcs(cb + 2 * cr + o, (uint8_t) (top >> 24));
    __stcs(cb + 2 * cr + o + a.pitch, (uint8_t) (bot >> 24));
    if (!(lane & 1)) {
        const uint32_t uv = export_cbcr<E>(export_block_straight(top, top1, bot, bot1));
        uint8_t* const pu = cb + (size_t) u * (a.pitch >> 1) + (X >> 1);
        __stcs(pu, (uint8_t) uv);
        __stcs(pu + cr, (uint8_t) (uv >> 8));
    }
}

template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) export_scaled_yuva_kernel(const __grid_constant__ ScaledArgs a) {
    const ExportFmt f = { Fmt, a.over, a.native, a.bg };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const uint32_t zc = f.over ? export_over(0u, f.bg, f.native) : 0u;   // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) (Fmt == GLAVA_B200_EXPORT_YUVA420P ? a.out_h >> 1 : a.out_h);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        scaled_yuva_item<false, E>(a, f, Fmt, rcp, zc, a.cr_offset, a.list + k, u, X, lane);
    }
}

template <typename Index>
static void launch_scaled_yuva(const ScaledArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.format == (GLAVA_B200_EXPORT_RGBA | GLB_EXPORT_STRAIGHT))
        export_scaled_yuva_kernel<Index, GLAVA_B200_EXPORT_RGBA | GLB_EXPORT_STRAIGHT, 0><<<blocks, 256, 0, st>>>(a);
    else if (a.format == (GLAVA_B200_EXPORT_BGRA | GLB_EXPORT_STRAIGHT))
        export_scaled_yuva_kernel<Index, GLAVA_B200_EXPORT_BGRA | GLB_EXPORT_STRAIGHT, 0><<<blocks, 256, 0, st>>>(a);
    else for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.format == GLAVA_B200_EXPORT_YUVA420P) export_scaled_yuva_kernel<Index, GLAVA_B200_EXPORT_YUVA420P, E><<<blocks, 256, 0, st>>>(a);
        else export_scaled_yuva_kernel<Index, GLAVA_B200_EXPORT_YUVA444P10, E><<<blocks, 256, 0, st>>>(a);
    });
}

// the scaled 10-bit kernels under an HDR encoding (DESIGN 4.22), as launch_hdr
template <typename Index, int E>
static void launch_scaled_hdr(const ScaledArgs& a, unsigned blocks, cudaStream_t st) {
    if (a.format == GLAVA_B200_EXPORT_P010) export_scaled_yuv_enc_kernel<Index, GLAVA_B200_EXPORT_P010, E><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV420P10) export_scaled_p10_kernel<Index, GLAVA_B200_EXPORT_YUV420P10, E><<<blocks, 256, 0, st>>>(a);
    else if (a.format == GLAVA_B200_EXPORT_YUV444P10) export_scaled_p10_kernel<Index, GLAVA_B200_EXPORT_YUV444P10, E><<<blocks, 256, 0, st>>>(a);
    else export_scaled_422_kernel<Index, GLAVA_B200_EXPORT_YUV422P10, E><<<blocks, 256, 0, st>>>(a);
}

int launch_export_scaled(const ScaledArgs& a, void* stream) {
    const uint64_t units = export_420(a.format) ? (uint64_t) (a.out_h >> 1) : (uint64_t) a.out_h;
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) ((a.out_w + 31) >> 5) * units);
    cudaStream_t st = (cudaStream_t) stream;
    if (a.enc >= GLB_ENC_PQ) {
        for_hdr(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (g.narrow) launch_scaled_hdr<uint32_t, E>(a, g.blocks, st);
            else launch_scaled_hdr<uint64_t, E>(a, g.blocks, st);
        });
        return launch_status("scaled export");
    }
    if (export_alpha(a.format)) {
        if (g.narrow) launch_scaled_yuva<uint32_t>(a, g.blocks, st);
        else launch_scaled_yuva<uint64_t>(a, g.blocks, st);
    } else if (export_422(a.format)) {
        if (g.narrow) launch_scaled_422<uint32_t>(a, g.blocks, st);
        else launch_scaled_422<uint64_t>(a, g.blocks, st);
    } else if (export_p10(a.format)) {
        if (g.narrow) launch_scaled_p10<uint32_t>(a, g.blocks, st);
        else launch_scaled_p10<uint64_t>(a, g.blocks, st);
    } else if (a.enc && a.format == GLAVA_B200_EXPORT_NV12) {
        for_enc(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (g.narrow) export_scaled_enc_kernel<uint32_t, E><<<g.blocks, 256, 0, st>>>(a);
            else export_scaled_enc_kernel<uint64_t, E><<<g.blocks, 256, 0, st>>>(a);
        });
    } else if (a.format != GLAVA_B200_EXPORT_NV12 && export_yuv(a.format)) {
        if (g.narrow) launch_scaled_yuv<uint32_t>(a, g.blocks, (cudaStream_t) stream);
        else launch_scaled_yuv<uint64_t>(a, g.blocks, (cudaStream_t) stream);
    } else if (g.narrow) export_scaled_kernel<uint32_t><<<g.blocks, 256, 0, (cudaStream_t) stream>>>(a);
    else export_scaled_kernel<uint64_t><<<g.blocks, 256, 0, (cudaStream_t) stream>>>(a);
    return launch_status("scaled export");
}

// ---- glava_b200_export_ladder (DESIGN 4.13) --------------------------------------------------------------------------------
// One warp per (entry, unit of the schedule), the unit fastest: a unit is one item of the rung's standalone kernel, run by
// that kernel's own body (export_item / scaled_item) with the rung's fields, so every rung is bit for bit its standalone
// call.  The schedule sorts one entry's units by the first source row they read, so the warps in flight cover a few source
// rows of one frame across all rungs; framebuffer loads keep normal L2 priority (Keep) for the rungs that follow.

// the fields export_item / scaled_item read, for one rung (named as ExportArgs / ScaledArgs name them)
struct RungView {
    const uint8_t*  fb;
    const uint32_t* marks;
    int mark_rows, w, h, format;
    size_t pitch;
    int src_x, src_y, src_w, src_h, out_w, out_h;
};

// One unit of export_ladder_enc_kernel: the item of rung g's standalone kernel under encoding E; Yuv as ladder_loop
template <bool Yuv, int E>
__device__ __forceinline__ void ladder_item(const LadderArgs& a, const LadderRung& g, const ExportEntryUV* e, int rung, int row,
                                            int col, int lane) {
    const RungView v = { a.fb, a.marks, a.mark_rows, a.w, a.h, g.format, g.pitch, g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h };
    const ExportFmt f = { g.format, g.over, a.native, g.bg };
    if (Yuv && g.format != GLAVA_B200_EXPORT_NV12 && export_yuv(g.format)) {
        const size_t cr = a.yuv[rung].cr_offset;
        if (g.whole) {
            const int x = col * 128 + lane * 4;
            if (x >= a.w) return;
            uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
            uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
            const int slot = __ldg(&e->slot);
            const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
            const ExportZero z = { a.yuv[rung].zy, a.yuv[rung].zu, a.yuv[rung].zv };
            yuv_item<true, E>(v, f, g.format, frame, slot, dst, cb, cr, row, col, x, z);
        } else {
            const ExportRecip rcp = { g.div_mul, g.div_shift };
            scaled_yuv_item<true, E>(v, f, g.format, rcp, g.zc, cr, e, row, col * 32 + lane, lane);
        }
    } else if (g.whole) {
        const int x = col * 128 + lane * 4;
        if (x >= a.w) return;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        // the entry's CbCr pointer as an offset from its luma (unsigned: the chroma may lie before it)
        const size_t uv_offset = g.format == GLAVA_B200_EXPORT_NV12
                                     ? (size_t) (__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)) - (unsigned long long) dst)
                                     : 0;
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        export_item<true, E>(v, f, frame, slot, dst, uv_offset, row, col, x, g.zy, g.zuv, g.zpx);
    } else {
        const ExportRecip rcp = { g.div_mul, g.div_shift };
        scaled_item<true, E>(v, f, rcp, g.zc, g.format == GLAVA_B200_EXPORT_NV12, e, row, col * 32 + lane, lane);
    }
}

// The ladder's loop; Yuv: the rungs may be I420, YUV444 or P010 (export_ladder_yuv_kernel), else they are NV12, RGBA or
// BGRA (export_ladder_kernel, whose code does not see the new formats).  Every rung is encoding 0.  ladder_item<Yuv, 0>
// written out: called, ptxas schedules the 64-bit index kernel differently, and these kernels keep their machine code.
template <typename Index, bool Yuv>
__device__ __forceinline__ void ladder_loop(const LadderArgs& a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const RungView v = { a.fb, a.marks, a.mark_rows, a.w, a.h, g.format, g.pitch, g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h };
        const ExportFmt f = { g.format, g.over, a.native, g.bg };
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (Yuv && g.format != GLAVA_B200_EXPORT_NV12 && export_yuv(g.format)) {
            const size_t cr = a.yuv[rung].cr_offset;
            if (g.whole) {
                const int x = col * 128 + lane * 4;
                if (x >= a.w) continue;
                uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
                uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
                const int slot = __ldg(&e->slot);
                const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
                const ExportZero z = { a.yuv[rung].zy, a.yuv[rung].zu, a.yuv[rung].zv };
                yuv_item<true>(v, f, g.format, frame, slot, dst, cb, cr, row, col, x, z);
            } else {
                const ExportRecip rcp = { g.div_mul, g.div_shift };
                scaled_yuv_item<true>(v, f, g.format, rcp, g.zc, cr, e, row, col * 32 + lane, lane);
            }
        } else if (g.whole) {
            const int x = col * 128 + lane * 4;
            if (x >= a.w) continue;
            uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
            // the entry's CbCr pointer as an offset from its luma (unsigned: the chroma may lie before it)
            const size_t uv_offset = g.format == GLAVA_B200_EXPORT_NV12
                                         ? (size_t) (__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)) - (unsigned long long) dst)
                                         : 0;
            const int slot = __ldg(&e->slot);
            const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
            export_item<true>(v, f, frame, slot, dst, uv_offset, row, col, x, g.zy, g.zuv, g.zpx);
        } else {
            const ExportRecip rcp = { g.div_mul, g.div_shift };
            scaled_item<true>(v, f, rcp, g.zc, g.format == GLAVA_B200_EXPORT_NV12, e, row, col * 32 + lane, lane);
        }
    }
}

// The loop of export_ladder_enc_kernel: any format and encoding per rung, each unit run by the instantiation of its rung's
template <typename Index>
__device__ __forceinline__ void ladder_enc_loop(const LadderArgs& a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (g.enc == 1) ladder_item<true, 1>(a, g, e, rung, row, col, lane);
        else if (g.enc == 2) ladder_item<true, 2>(a, g, e, rung, row, col, lane);
        else if (g.enc == 3) ladder_item<true, 3>(a, g, e, rung, row, col, lane);
        else ladder_item<true, 0>(a, g, e, rung, row, col, lane);
    }
}

template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_kernel(const __grid_constant__ LadderArgs a) { ladder_loop<Index, false>(a); }
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_yuv_kernel(const __grid_constant__ LadderArgs a) { ladder_loop<Index, true>(a); }
// any format and encoding per rung (DESIGN 4.15)
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_enc_kernel(const __grid_constant__ LadderArgs a) { ladder_enc_loop<Index>(a); }

// One unit of a planar 10-bit rung of export_ladder_p10_kernel under encoding E: the item of its standalone kernel
// (export_p10_kernel / export_scaled_p10_kernel), as ladder_item runs the other Y'CbCr rungs
template <int E>
__device__ __forceinline__ void ladder_p10_item(const LadderArgs& a, const LadderRung& g, const ExportEntryUV* e, int rung, int row,
                                                int col, int lane) {
    const RungView v = { a.fb, a.marks, a.mark_rows, a.w, a.h, g.format, g.pitch, g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h };
    const ExportFmt f = { g.format, g.over, a.native, g.bg };
    const size_t cr = a.yuv[rung].cr_offset;
    if (g.whole) {
        const int x = col * 128 + lane * 4;
        if (x >= a.w) return;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        const ExportZero z = { a.yuv[rung].zy, a.yuv[rung].zu, a.yuv[rung].zv };
        p10_item<true, E>(v, f, g.format, frame, slot, dst, cb, cr, row, col, x, z);
    } else {
        const ExportRecip rcp = { g.div_mul, g.div_shift };
        scaled_p10_item<true, E>(v, f, g.format, rcp, g.zc, cr, e, row, col * 32 + lane, lane);
    }
}

// Any format and encoding per rung, launched only when a rung is YUV420P10 or YUV444P10 (DESIGN 4.16): planar 10-bit
// units run ladder_p10_item, the others ladder_item, each in its rung's encoding
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_p10_kernel(const __grid_constant__ LadderArgs a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (export_p10(g.format)) {
            if (g.enc == 1) ladder_p10_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_p10_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_p10_item<3>(a, g, e, rung, row, col, lane);
            else ladder_p10_item<0>(a, g, e, rung, row, col, lane);
        } else if (g.enc == 1) ladder_item<true, 1>(a, g, e, rung, row, col, lane);
        else if (g.enc == 2) ladder_item<true, 2>(a, g, e, rung, row, col, lane);
        else if (g.enc == 3) ladder_item<true, 3>(a, g, e, rung, row, col, lane);
        else ladder_item<true, 0>(a, g, e, rung, row, col, lane);
    }
}

// One unit of a 4:2:2 rung of export_ladder_422_kernel under encoding E: the item of its standalone kernel
// (export_422_kernel / export_scaled_422_kernel), as ladder_p10_item
template <int E>
__device__ __forceinline__ void ladder_422_item(const LadderArgs& a, const LadderRung& g, const ExportEntryUV* e, int rung, int row,
                                                int col, int lane) {
    const RungView v = { a.fb, a.marks, a.mark_rows, a.w, a.h, g.format, g.pitch, g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h };
    const ExportFmt f = { g.format, g.over, a.native, g.bg };
    const size_t cr = a.yuv[rung].cr_offset;
    if (g.whole) {
        const int x = col * 128 + lane * 4;
        if (x >= a.w) return;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        const ExportZero z = { a.yuv[rung].zy, a.yuv[rung].zu, a.yuv[rung].zv };
        item_422<true, E>(v, f, g.format, frame, slot, dst, cb, cr, row, col, x, z);
    } else {
        const ExportRecip rcp = { g.div_mul, g.div_shift };
        scaled_422_item<true, E>(v, f, g.format, rcp, g.zc, cr, e, row, col * 32 + lane, lane);
    }
}

// Any format and encoding per rung, launched only when a rung is YUV422P, YUV422P10 or UYVY (DESIGN 4.18): 4:2:2 units run
// ladder_422_item, planar 10-bit units ladder_p10_item, the others ladder_item, each in its rung's encoding, so that
// export_ladder_p10_kernel and the older ladder kernels keep their machine code
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_422_kernel(const __grid_constant__ LadderArgs a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (export_422(g.format)) {
            if (g.enc == 1) ladder_422_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_422_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_422_item<3>(a, g, e, rung, row, col, lane);
            else ladder_422_item<0>(a, g, e, rung, row, col, lane);
        } else if (export_p10(g.format)) {
            if (g.enc == 1) ladder_p10_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_p10_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_p10_item<3>(a, g, e, rung, row, col, lane);
            else ladder_p10_item<0>(a, g, e, rung, row, col, lane);
        } else if (g.enc == 1) ladder_item<true, 1>(a, g, e, rung, row, col, lane);
        else if (g.enc == 2) ladder_item<true, 2>(a, g, e, rung, row, col, lane);
        else if (g.enc == 3) ladder_item<true, 3>(a, g, e, rung, row, col, lane);
        else ladder_item<true, 0>(a, g, e, rung, row, col, lane);
    }
}

// One unit of an alpha rung of export_ladder_yuva_kernel under encoding E: the item of its standalone kernel
// (export_yuva_kernel / export_scaled_yuva_kernel), as ladder_p10_item; yuv[rung].za is what a zero pixel's A becomes
template <int E>
__device__ __forceinline__ void ladder_yuva_item(const LadderArgs& a, const LadderRung& g, const ExportEntryUV* e, int rung, int row,
                                                 int col, int lane) {
    const RungView v = { a.fb, a.marks, a.mark_rows, a.w, a.h, g.format, g.pitch, g.src_x, g.src_y, g.src_w, g.src_h, g.out_w, g.out_h };
    const ExportFmt f = { g.format, g.over, a.native, g.bg };
    const size_t cr = a.yuv[rung].cr_offset;
    if (g.whole) {
        const int x = col * 128 + lane * 4;
        if (x >= a.w) return;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        uint8_t* const cb = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        const ExportZeroA z = { a.yuv[rung].zy, a.yuv[rung].zu, a.yuv[rung].zv, a.yuv[rung].za };
        yuva_item<true, E>(v, f, g.format, frame, slot, dst, cb, cr, row, col, x, z);
    } else {
        const ExportRecip rcp = { g.div_mul, g.div_shift };
        scaled_yuva_item<true, E>(v, f, g.format, rcp, g.zc, cr, e, row, col * 32 + lane, lane);
    }
}

// Any format and encoding per rung, launched only when a rung is YUVA420P, YUVA444P10 or straight RGBA / BGRA (DESIGN
// 4.19): alpha units run ladder_yuva_item, 4:2:2 units ladder_422_item, planar 10-bit units ladder_p10_item, the others
// ladder_item, each in its rung's encoding, so that the older ladder kernels keep their machine code
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_yuva_kernel(const __grid_constant__ LadderArgs a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (export_alpha(g.format)) {
            if (g.enc == 1) ladder_yuva_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_yuva_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_yuva_item<3>(a, g, e, rung, row, col, lane);
            else ladder_yuva_item<0>(a, g, e, rung, row, col, lane);
        } else if (export_422(g.format)) {
            if (g.enc == 1) ladder_422_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_422_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_422_item<3>(a, g, e, rung, row, col, lane);
            else ladder_422_item<0>(a, g, e, rung, row, col, lane);
        } else if (export_p10(g.format)) {
            if (g.enc == 1) ladder_p10_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_p10_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_p10_item<3>(a, g, e, rung, row, col, lane);
            else ladder_p10_item<0>(a, g, e, rung, row, col, lane);
        } else if (g.enc == 1) ladder_item<true, 1>(a, g, e, rung, row, col, lane);
        else if (g.enc == 2) ladder_item<true, 2>(a, g, e, rung, row, col, lane);
        else if (g.enc == 3) ladder_item<true, 3>(a, g, e, rung, row, col, lane);
        else ladder_item<true, 0>(a, g, e, rung, row, col, lane);
    }
}

// One unit of export_ladder_hdr_kernel under the HDR encoding E (DESIGN 4.22): the item of its rung's standalone kernel
// (P010: export_yuv_enc_kernel's; the planar 10-bit formats: export_p10_kernel's; YUV422P10: export_422_kernel's, or their
// scaled forms) in that kernel's HDR instantiation
template <int E>
__device__ __forceinline__ void ladder_hdr_item(const LadderArgs& a, const LadderRung& g, const ExportEntryUV* e, int rung, int row,
                                                int col, int lane) {
    if (export_422(g.format)) ladder_422_item<E>(a, g, e, rung, row, col, lane);
    else if (export_p10(g.format)) ladder_p10_item<E>(a, g, e, rung, row, col, lane);
    else ladder_item<true, E>(a, g, e, rung, row, col, lane);
}

// Any format and encoding per rung, launched only when a rung is HDR (DESIGN 4.22): HDR units run ladder_hdr_item, every
// other unit what export_ladder_yuva_kernel runs for it, so that HDR and SDR rungs mix in one launch and the older ladder
// kernels keep their machine code
template <typename Index>
__global__ void __launch_bounds__(256) export_ladder_hdr_kernel(const __grid_constant__ LadderArgs a) {
    const Index units = (Index) a.units, items = (Index) a.count * units;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / units;
        const uint64_t unit = __ldg(reinterpret_cast<const unsigned long long*>(a.sched) + (it - k * units));
        const int rung = ladder_unit_rung(unit), row = ladder_unit_row(unit), col = ladder_unit_col(unit);
        const LadderRung& g = a.rung[rung];
        const ExportEntryUV* e = a.list + (size_t) k * a.nrungs + rung;
        if (g.enc == GLB_ENC_PQ) ladder_hdr_item<GLB_ENC_PQ>(a, g, e, rung, row, col, lane);
        else if (g.enc == GLB_ENC_HLG) ladder_hdr_item<GLB_ENC_HLG>(a, g, e, rung, row, col, lane);
        else if (export_alpha(g.format)) {
            if (g.enc == 1) ladder_yuva_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_yuva_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_yuva_item<3>(a, g, e, rung, row, col, lane);
            else ladder_yuva_item<0>(a, g, e, rung, row, col, lane);
        } else if (export_422(g.format)) {
            if (g.enc == 1) ladder_422_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_422_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_422_item<3>(a, g, e, rung, row, col, lane);
            else ladder_422_item<0>(a, g, e, rung, row, col, lane);
        } else if (export_p10(g.format)) {
            if (g.enc == 1) ladder_p10_item<1>(a, g, e, rung, row, col, lane);
            else if (g.enc == 2) ladder_p10_item<2>(a, g, e, rung, row, col, lane);
            else if (g.enc == 3) ladder_p10_item<3>(a, g, e, rung, row, col, lane);
            else ladder_p10_item<0>(a, g, e, rung, row, col, lane);
        } else if (g.enc == 1) ladder_item<true, 1>(a, g, e, rung, row, col, lane);
        else if (g.enc == 2) ladder_item<true, 2>(a, g, e, rung, row, col, lane);
        else if (g.enc == 3) ladder_item<true, 3>(a, g, e, rung, row, col, lane);
        else ladder_item<true, 0>(a, g, e, rung, row, col, lane);
    }
}

int launch_export_ladder(const LadderArgs& a, void* stream) {
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) a.units);
    int format[GLAVA_B200_LADDER_MAX], enc[GLAVA_B200_LADDER_MAX];
    for (int j = 0; j < a.nrungs; ++j) { format[j] = a.rung[j].format; enc[j] = a.rung[j].enc; }
    const int kind = ladder_kernel(format, enc, a.nrungs);
    cudaStream_t st = (cudaStream_t) stream;
    if (kind == ladder_hdr) {
        if (g.narrow) export_ladder_hdr_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_hdr_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (kind == ladder_yuva) {
        if (g.narrow) export_ladder_yuva_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_yuva_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (kind == ladder_422) {
        if (g.narrow) export_ladder_422_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_422_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (kind == ladder_p10) {
        if (g.narrow) export_ladder_p10_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_p10_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (kind == ladder_enc) {
        if (g.narrow) export_ladder_enc_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_enc_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (kind == ladder_yuv) {
        if (g.narrow) export_ladder_yuv_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
        else export_ladder_yuv_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    } else if (g.narrow) export_ladder_kernel<uint32_t><<<g.blocks, 256, 0, st>>>(a);
    else export_ladder_kernel<uint64_t><<<g.blocks, 256, 0, st>>>(a);
    return launch_status("ladder export");
}

// ---- glava_b200_overlay_frames (DESIGN 4.12) -------------------------------------------------------------------------------
// Native opacity: a quad of four framebuffer pixels that is not all zero is loaded together with the destination bytes under
// it, blended (export_core.h overlay_px / overlay_nv12_quad) and stored back; an all-zero quad touches nothing.  With marks
// the items are bands (Band = true): one warp per (entry, band of mark_rows rows, strip); a band whose word is empty costs
// that word, otherwise only its marked rows are visited (NV12: the row pairs overlay_band_pairs gives it).  Without marks,
// and under any other opacity (the rectangle then gets export_kernel's opaque bytes, every row), one warp per (entry, output
// row pair, strip) as export_kernel.  A lane owns a quad; widths that are not a multiple of 4 take a per-pixel tail.

// native RGBA / BGRA: the quad at x of one destination row
__device__ __forceinline__ void overlay_rgba(uint8_t* row, int x, int w, bool bgra, const uint32_t in[4]) {
    if ((in[0] | in[1] | in[2] | in[3]) == 0u) return;
    uint32_t px[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) px[k] = bgra ? export_swap_rb(in[k]) : in[k];
    uint32_t* out = reinterpret_cast<uint32_t*>(row) + x;
    if (x + 4 <= w) {                                       // dst and pitch: multiples of 16
        uint4 d = __ldcs(reinterpret_cast<const uint4*>(out));
        d.x = overlay_px(px[0], d.x); d.y = overlay_px(px[1], d.y); d.z = overlay_px(px[2], d.z); d.w = overlay_px(px[3], d.w);
        __stcs(reinterpret_cast<uint4*>(out), d);
    } else {
        for (int k = 0; k < 4 && x + k < w; ++k) __stcs(out + k, overlay_px(px[k], __ldcs(out + k)));
    }
}

// NV12 of the quad at x of output rows 2j, 2j + 1 (r0: row 2j's Y bytes, uv: the pair's CbCr row); native: blended onto the
// bytes there, skipped when all eight pixels are zero; otherwise export_kernel's bytes (f: composite, opacity not native).
// E: the destination's encoding.
template <int E>
__device__ __forceinline__ void overlay_nv12(const ExportFmt& f, bool native, uint8_t* r0, uint8_t* uv, size_t pitch, int x, int w,
                                             const uint32_t top[4], const uint32_t bot[4]) {
    const bool full = x + 4 <= w;                           // else w even: the last two pixels of a row
    uint32_t yt, yb, c;
    if (native) {
        if ((top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) == 0u) return;
        if (full) {
            yt = __ldcs(reinterpret_cast<const uint32_t*>(r0 + x));
            yb = __ldcs(reinterpret_cast<const uint32_t*>(r0 + pitch + x));
            c = __ldcs(reinterpret_cast<const uint32_t*>(uv + x));
        } else {
            yt = __ldcs(reinterpret_cast<const unsigned short*>(r0 + x));
            yb = __ldcs(reinterpret_cast<const unsigned short*>(r0 + pitch + x));
            c = __ldcs(reinterpret_cast<const unsigned short*>(uv + x));
        }
        overlay_nv12_quad<E>(top, bot, &yt, &yb, &c);
    } else {
        c = export_nv12_quad<E>(f, top, bot, &yt, &yb);
    }
    if (full) {
        __stcs(reinterpret_cast<uint32_t*>(r0 + x), yt);
        __stcs(reinterpret_cast<uint32_t*>(r0 + pitch + x), yb);
        __stcs(reinterpret_cast<uint32_t*>(uv + x), c);
    } else {
        __stcs(reinterpret_cast<unsigned short*>(r0 + x), (unsigned short) yt);
        __stcs(reinterpret_cast<unsigned short*>(r0 + pitch + x), (unsigned short) yb);
        __stcs(reinterpret_cast<unsigned short*>(uv + x), (unsigned short) c);
    }
}

template <typename A>
__device__ __forceinline__ uint32_t overlay_mark(const A& a, int slot, int y, int strip) {
    return __ldg(a.marks + export_mark_index(slot, a.w, a.h, a.mark_rows, y, strip));
}

// The walk of overlay_loop below (its items and mark-aware reads) with what a format does to the destination left to Body,
// for glava_b200_overlay_planes (DESIGN 4.17).  overlay_loop keeps its own written-out copy: run through this template,
// ptxas orders the row-pair item's blocks differently, and overlay_kernel / overlay_enc_kernel keep their machine code.
// Body (the destination of one entry):
//   b.a                       the argument struct (fb, marks, mark_rows, list, count, w, h)
//   Body::dst(e)              the entry's first plane
//   b.pairs()                 band items walk output row pairs (4:2:0), else output rows
//   b.row(e, dst, r, x, q)    native: the quad q at x onto output row r
//   b.chroma(e)               the entry's chroma, loaded once per band item that walks pairs
//   b.pair(dst, c, j, x, t, b)  native: the quads of output rows 2j and 2j + 1
//   b.item(e, dst, u, x, t, b, y1)   a row-pair item: output rows 2u and 2u + 1 (framebuffer row y1 >= 0), any opacity
template <typename Index, bool Band, typename Body>
__device__ __forceinline__ void overlay_walk(const Body& b) {
    const auto& a = b.a;
    const int rows = Band ? a.mark_rows : 2;
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + rows - 1) / rows);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / strips), strip = (int) (rem - (Index) u * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const auto* e = a.list + k;
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        uint8_t* const dst = Body::dst(e);
        if (Band) {                                         // native, marks: band u
            const int b0 = u * rows, b1 = min(b0 + rows, a.h);
            const uint32_t mark = overlay_mark(a, slot, b0, strip);
            const int lo = max((int) (mark & 0xffffu), b0), hi = min((int) (mark >> 16), b1);
            if (lo >= hi) continue;
            if (!b.pairs()) {
                for (int y = lo; y < hi; ++y) {
                    uint32_t q[4];
                    load_quad(frame, a.w, y, x, q);
                    b.row(e, dst, a.h - 1 - y, x, q);
                }
                continue;
            }
            const auto c = b.chroma(e);
            int ja, jb;
            const uint32_t below = overlay_band_pairs(a.h, b0, lo, hi, &ja, &jb) ? overlay_mark(a, slot, b0 - 1, strip) : 0u;
            if (overlay_top_straddles(a.h, b1, ja) && export_row_read(overlay_mark(a, slot, b1, strip), b1)) ++ja;
            for (int j = ja; j < jb; ++j) {
                const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
                uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
                if (y0 >= lo && y0 < hi) load_quad(frame, a.w, y0, x, top);
                if (y1 >= b0 ? y1 >= lo && y1 < hi : export_row_read(below, y1)) load_quad(frame, a.w, y1, x, bot);
                b.pair(dst, c, j, x, top, bot);
            }
        } else {                                            // output rows 2u, 2u + 1: framebuffer rows y0, y0 - 1
            const int y0 = a.h - 1 - 2 * u, y1 = y0 - 1;
            uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
            if (!a.marks || export_row_read(overlay_mark(a, slot, y0, strip), y0)) load_quad(frame, a.w, y0, x, top);
            if (y1 >= 0 && (!a.marks || export_row_read(overlay_mark(a, slot, y1, strip), y1))) load_quad(frame, a.w, y1, x, bot);
            b.item(e, dst, u, x, top, bot, y1);
        }
    }
}

template <typename Index, bool Band, int E>
__device__ __forceinline__ void overlay_loop(const OverlayArgs& a) {
    const ExportFmt f = { a.format, 1, 0, 0u };             // any other opacity: the stored colour, alpha 255
    const bool nv12 = a.format == GLAVA_B200_EXPORT_NV12, bgra = a.format == GLAVA_B200_EXPORT_BGRA;
    const int rows = Band ? a.mark_rows : 2;
    const Index strips = (Index) ((a.w + 127) >> 7), per = strips * (Index) ((a.h + rows - 1) / rows);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / strips), strip = (int) (rem - (Index) u * strips);
        const int x = strip * 128 + lane * 4;
        if (x >= a.w) continue;
        const ExportEntryUV* e = a.list + k;
        const int slot = __ldg(&e->slot);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        uint8_t* const dst = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
        if (Band) {                                         // native, marks: band u
            const int b0 = u * rows, b1 = min(b0 + rows, a.h);
            const uint32_t mark = overlay_mark(a, slot, b0, strip);
            const int lo = max((int) (mark & 0xffffu), b0), hi = min((int) (mark >> 16), b1);
            if (lo >= hi) continue;
            if (!nv12) {
                for (int y = lo; y < hi; ++y) {
                    uint32_t q[4];
                    load_quad(frame, a.w, y, x, q);
                    overlay_rgba(dst + (size_t) (a.h - 1 - y) * a.pitch, x, a.w, bgra, q);
                }
                continue;
            }
            uint8_t* const dst_uv = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
            int ja, jb;
            const uint32_t below = overlay_band_pairs(a.h, b0, lo, hi, &ja, &jb) ? overlay_mark(a, slot, b0 - 1, strip) : 0u;
            if (overlay_top_straddles(a.h, b1, ja) && export_row_read(overlay_mark(a, slot, b1, strip), b1)) ++ja;
            for (int j = ja; j < jb; ++j) {
                const int y0 = a.h - 1 - 2 * j, y1 = y0 - 1;
                uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
                if (y0 >= lo && y0 < hi) load_quad(frame, a.w, y0, x, top);
                if (y1 >= b0 ? y1 >= lo && y1 < hi : export_row_read(below, y1)) load_quad(frame, a.w, y1, x, bot);
                overlay_nv12<E>(f, true, dst + (size_t) (2 * j) * a.pitch, dst_uv + (size_t) j * a.pitch, a.pitch, x, a.w, top, bot);
            }
        } else {                                            // output rows 2u, 2u + 1: framebuffer rows y0, y0 - 1
            const int y0 = a.h - 1 - 2 * u, y1 = y0 - 1;
            uint32_t top[4] = { 0u, 0u, 0u, 0u }, bot[4] = { 0u, 0u, 0u, 0u };
            if (!a.marks || export_row_read(overlay_mark(a, slot, y0, strip), y0)) load_quad(frame, a.w, y0, x, top);
            if (y1 >= 0 && (!a.marks || export_row_read(overlay_mark(a, slot, y1, strip), y1))) load_quad(frame, a.w, y1, x, bot);
            uint8_t* const r0 = dst + (size_t) (2 * u) * a.pitch;
            if (nv12) {
                uint8_t* const dst_uv = reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
                overlay_nv12<E>(f, a.native, r0, dst_uv + (size_t) u * a.pitch, a.pitch, x, a.w, top, bot);
            } else if (a.native) {
                overlay_rgba(r0, x, a.w, bgra, top);
                if (y1 >= 0) overlay_rgba(r0 + a.pitch, x, a.w, bgra, bot);
            } else {
                store_rgba(f, r0, x, a.w, top, export_px(f, 0u));
                if (y1 >= 0) store_rgba(f, r0 + a.pitch, x, a.w, bot, export_px(f, 0u));
            }
        }
    }
}

template <typename Index, bool Band>
__global__ void __launch_bounds__(256) overlay_kernel(const __grid_constant__ OverlayArgs a) { overlay_loop<Index, Band, 0>(a); }
// NV12 destinations in encoding E = 1..3
template <typename Index, bool Band, int E>
__global__ void __launch_bounds__(256) overlay_enc_kernel(const __grid_constant__ OverlayArgs a) { overlay_loop<Index, Band, E>(a); }

static void launch_overlay_fade(const OverlayArgs& a, const ExportGrid& g, cudaStream_t st);   // DESIGN 4.20, below

int launch_overlay(const OverlayArgs& a, void* stream) {
    const int rows = a.band ? a.mark_rows : 2;
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) ((a.w + 127) >> 7) * (uint64_t) ((a.h + rows - 1) / rows));
    cudaStream_t st = (cudaStream_t) stream;
    if (a.fade) {
        launch_overlay_fade(a, g, st);
    } else if (a.enc) {
        for_enc(a.enc, [&](auto e) {
            constexpr int E = decltype(e)::value;
            if (a.band) {
                if (g.narrow) overlay_enc_kernel<uint32_t, true, E><<<g.blocks, 256, 0, st>>>(a);
                else overlay_enc_kernel<uint64_t, true, E><<<g.blocks, 256, 0, st>>>(a);
            } else {
                if (g.narrow) overlay_enc_kernel<uint32_t, false, E><<<g.blocks, 256, 0, st>>>(a);
                else overlay_enc_kernel<uint64_t, false, E><<<g.blocks, 256, 0, st>>>(a);
            }
        });
    } else if (a.band) {
        if (g.narrow) overlay_kernel<uint32_t, true><<<g.blocks, 256, 0, st>>>(a);
        else overlay_kernel<uint64_t, true><<<g.blocks, 256, 0, st>>>(a);
    } else {
        if (g.narrow) overlay_kernel<uint32_t, false><<<g.blocks, 256, 0, st>>>(a);
        else overlay_kernel<uint64_t, false><<<g.blocks, 256, 0, st>>>(a);
    }
    return launch_status("overlay");
}

// ---- glava_b200_overlay_planes (DESIGN 4.17) -------------------------------------------------------------------------------
// overlay_walk onto decoded pictures: per entry three plane pointers (OverlayPlanesEntry), one luma pitch and one
// chroma pitch per call.  NV12 runs overlay_frames' own item body (overlay_nv12); I420, P010 and YUV420P10 walk row pairs as
// NV12 does; YUV444 and YUV444P10 walk rows as RGBA does.  Native opacity blends (export_core.h overlay_*_quad) and leaves
// all-zero quads alone; any other opacity writes export_frames' bytes of the format.  Tails: the last two pixels of a row
// for the 4:2:0 formats (w even), sample by sample for the 4:4:4 ones.  One kernel per format and encoding.  The 4:2:2
// formats (DESIGN 4.18) walk rows through row422, each row's pixel pairs blended as 4:2:0 blocks of that pair, w even.

// the first n (1..4) bytes at p as a word (n == 4: p is 4-byte aligned)
__device__ __forceinline__ uint32_t load_bytes(const uint8_t* p, int n) {
    if (n >= 4) return __ldcs(reinterpret_cast<const uint32_t*>(p));
    uint32_t v = 0u;
    for (int k = 0; k < n; ++k) v |= (uint32_t) __ldcs(p + k) << (8 * k);
    return v;
}
// the first n (1..4) uint16 samples at p as two words (n == 4: p is 8-byte aligned); as store_u16, written out
__device__ __forceinline__ void load_u16(const uint8_t* p, uint32_t v[2], int n) {
    if (n >= 4) {
        const uint2 d = __ldcs(reinterpret_cast<const uint2*>(p));
        v[0] = d.x; v[1] = d.y;
        return;
    }
    const unsigned short* const q = reinterpret_cast<const unsigned short*>(p);
    v[0] = __ldcs(q); v[1] = 0u;
    if (n > 1) v[0] |= (uint32_t) __ldcs(q + 1) << 16;
    if (n > 2) v[1] = __ldcs(q + 2);
}

template <int Fmt, int E>
struct OverlayPlanesBody {
    static constexpr bool k420 = Fmt == GLAVA_B200_EXPORT_NV12 || Fmt == GLAVA_B200_EXPORT_I420 || Fmt == GLAVA_B200_EXPORT_P010 ||
                                 Fmt == GLAVA_B200_EXPORT_YUV420P10;
    static constexpr bool kPlanar = Fmt == GLAVA_B200_EXPORT_I420 || Fmt == GLAVA_B200_EXPORT_YUV444 || Fmt == GLAVA_B200_EXPORT_YUV420P10 ||
                                    Fmt == GLAVA_B200_EXPORT_YUV444P10 || Fmt == GLAVA_B200_EXPORT_YUV422P ||
                                    Fmt == GLAVA_B200_EXPORT_YUV422P10;
    // 4:2:2 (DESIGN 4.18) walks rows as 4:4:4 does, through row422; UYVY has no chroma plane
    static constexpr bool k422 = Fmt == GLAVA_B200_EXPORT_YUV422P || Fmt == GLAVA_B200_EXPORT_YUV422P10 || Fmt == GLAVA_B200_EXPORT_UYVY;
    struct Chroma { uint8_t* cb; uint8_t* cr; };
    const OverlayPlanesArgs& a;
    ExportFmt f;                                            // any other opacity: the stored colour, alpha 255
    __device__ __forceinline__ explicit OverlayPlanesBody(const OverlayPlanesArgs& a_) : a(a_), f{ Fmt, 1, 0, 0u } {}
    static __device__ __forceinline__ uint8_t* plane(const OverlayPlanesEntry* e, int p) {
        return reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->plane[p])));
    }
    static __device__ __forceinline__ uint8_t* dst(const OverlayPlanesEntry* e) { return plane(e, 0); }
    __device__ __forceinline__ bool pairs() const { return k420; }
    __device__ __forceinline__ Chroma chroma(const OverlayPlanesEntry* e) const {
        if constexpr (Fmt == GLAVA_B200_EXPORT_UYVY) return { nullptr, nullptr };
        else return { plane(e, 1), kPlanar ? plane(e, 2) : nullptr };
    }

    // 4:4:4: the quad at x of output row r (native: blended, all zero: untouched)
    __device__ __forceinline__ void row444(bool native, uint8_t* dst, Chroma c, int r, int x, const uint32_t q[4]) const {
        if (native && (q[0] | q[1] | q[2] | q[3]) == 0u) return;
        const int n = x + 4 <= a.w ? 4 : a.w - x;
        if (Fmt == GLAVA_B200_EXPORT_YUV444) {
            uint8_t* const py = dst + (size_t) r * a.pitch + x;
            uint8_t* const pu = c.cb + (size_t) r * a.chroma_pitch + x;
            uint8_t* const pv = c.cr + (size_t) r * a.chroma_pitch + x;
            uint32_t y, u, v;
            if (native) {
                y = load_bytes(py, n); u = load_bytes(pu, n); v = load_bytes(pv, n);
                overlay_444_quad<E>(q, &y, &u, &v);
            } else {
                export_444_quad<E>(f, q, &y, &u, &v);
            }
            store_bytes(py, y, n); store_bytes(pu, u, n); store_bytes(pv, v, n);
        } else {                                            // YUV444P10
            uint8_t* const py = dst + (size_t) r * a.pitch + 2 * (size_t) x;
            uint8_t* const pu = c.cb + (size_t) r * a.chroma_pitch + 2 * (size_t) x;
            uint8_t* const pv = c.cr + (size_t) r * a.chroma_pitch + 2 * (size_t) x;
            uint32_t y[2], u[2], v[2];
            if (native) {
                load_u16(py, y, n); load_u16(pu, u, n); load_u16(pv, v, n);
                overlay_444p10_quad<E>(q, y, u, v);
            } else {
                export_444p10_quad<E>(f, q, y, u, v);
            }
            store_u16(py, y, n); store_u16(pu, u, n); store_u16(pv, v, n);
        }
    }
    // 4:2:0: the quads at x of output rows 2j and 2j + 1 (native: blended, all eight pixels zero: untouched)
    __device__ __forceinline__ void pair420(bool native, uint8_t* dst, Chroma c, int j, int x, const uint32_t top[4],
                                            const uint32_t bot[4]) const {
        uint8_t* const r0 = dst + (size_t) (2 * j) * a.pitch;
        uint8_t* const cj = c.cb + (size_t) j * a.chroma_pitch;
        if (Fmt == GLAVA_B200_EXPORT_NV12) {
            overlay_nv12<E>(f, native, r0, cj, a.pitch, x, a.w, top, bot);
            return;
        }
        if (native && (top[0] | top[1] | top[2] | top[3] | bot[0] | bot[1] | bot[2] | bot[3]) == 0u) return;
        const bool full = x + 4 <= a.w;                     // else w even: the last two pixels of a row
        if (Fmt == GLAVA_B200_EXPORT_I420) {
            uint8_t* const pu = cj + (x >> 1);
            uint8_t* const pv = c.cr + (size_t) j * a.chroma_pitch + (x >> 1);
            uint32_t yt, yb, u, v;
            if (native) {
                yt = load_bytes(r0 + x, full ? 4 : 2); yb = load_bytes(r0 + a.pitch + x, full ? 4 : 2);
                u = load_bytes(pu, full ? 2 : 1); v = load_bytes(pv, full ? 2 : 1);
                overlay_i420_quad<E>(top, bot, &yt, &yb, &u, &v);
            } else {
                const uint32_t uv = export_nv12_quad<E>(f, top, bot, &yt, &yb);
                u = export_cb_pair(uv); v = export_cr_pair(uv);
            }
            if (full) {
                __stcs(reinterpret_cast<uint32_t*>(r0 + x), yt);
                __stcs(reinterpret_cast<uint32_t*>(r0 + a.pitch + x), yb);
                __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u);
                __stcs(reinterpret_cast<unsigned short*>(pv), (unsigned short) v);
            } else {
                __stcs(reinterpret_cast<unsigned short*>(r0 + x), (unsigned short) yt);
                __stcs(reinterpret_cast<unsigned short*>(r0 + a.pitch + x), (unsigned short) yb);
                __stcs(pu, (uint8_t) u);
                __stcs(pv, (uint8_t) v);
            }
            return;
        }
        // P010: chroma words (Cb, Cr) per block at cj + 2x; YUV420P10: two Cb samples at cj + x, two Cr samples in the Cr plane
        constexpr bool msb = Fmt == GLAVA_B200_EXPORT_P010;
        uint8_t* const py = r0 + 2 * (size_t) x;
        uint8_t* const pu = msb ? cj + 2 * (size_t) x : cj + x;
        uint8_t* const pv = msb ? nullptr : c.cr + (size_t) j * a.chroma_pitch + x;
        uint32_t yt[2] = { 0u, 0u }, yb[2] = { 0u, 0u }, uv[2] = { 0u, 0u };
        if (native) {
            if (full) {
                const uint2 t = __ldcs(reinterpret_cast<const uint2*>(py)), b = __ldcs(reinterpret_cast<const uint2*>(py + a.pitch));
                yt[0] = t.x; yt[1] = t.y; yb[0] = b.x; yb[1] = b.y;
                if (msb) {
                    const uint2 d = __ldcs(reinterpret_cast<const uint2*>(pu));
                    uv[0] = d.x; uv[1] = d.y;
                } else {
                    uv[0] = __ldcs(reinterpret_cast<const uint32_t*>(pu)); uv[1] = __ldcs(reinterpret_cast<const uint32_t*>(pv));
                }
            } else {
                yt[0] = __ldcs(reinterpret_cast<const uint32_t*>(py)); yb[0] = __ldcs(reinterpret_cast<const uint32_t*>(py + a.pitch));
                if (msb) uv[0] = __ldcs(reinterpret_cast<const uint32_t*>(pu));
                else { uv[0] = __ldcs(reinterpret_cast<const unsigned short*>(pu)); uv[1] = __ldcs(reinterpret_cast<const unsigned short*>(pv)); }
            }
            overlay_p10_quad<E, msb>(top, bot, yt, yb, uv);
        } else if (msb) {
            export_p010_quad<E>(f, top, bot, yt, yb, uv);
        } else {
            export_i010_quad<E>(f, top, bot, yt, yb, &uv[0], &uv[1]);
        }
        if (full) {
            __stcs(reinterpret_cast<uint2*>(py), make_uint2(yt[0], yt[1]));
            __stcs(reinterpret_cast<uint2*>(py + a.pitch), make_uint2(yb[0], yb[1]));
            if (msb) __stcs(reinterpret_cast<uint2*>(pu), make_uint2(uv[0], uv[1]));
            else { __stcs(reinterpret_cast<uint32_t*>(pu), uv[0]); __stcs(reinterpret_cast<uint32_t*>(pv), uv[1]); }
        } else {
            __stcs(reinterpret_cast<uint32_t*>(py), yt[0]);
            __stcs(reinterpret_cast<uint32_t*>(py + a.pitch), yb[0]);
            if (msb) __stcs(reinterpret_cast<uint32_t*>(pu), uv[0]);
            else { __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) uv[0]); __stcs(reinterpret_cast<unsigned short*>(pv), (unsigned short) uv[1]); }
        }
    }

    // 4:2:2: the quad at x of output row r (native: blended, all zero: untouched); w even, so past the last full quad the
    // last pixel pair of a row
    __device__ __forceinline__ void row422(bool native, uint8_t* dst, Chroma c, int r, int x, const uint32_t q[4]) const {
        if (native && (q[0] | q[1] | q[2] | q[3]) == 0u) return;
        const bool full = x + 4 <= a.w;
        if (Fmt == GLAVA_B200_EXPORT_UYVY) {
            uint8_t* const p = dst + (size_t) r * a.pitch + 2 * (size_t) x;
            uint32_t w[2] = { 0u, 0u }, y, uv;
            if (native) {
                if (full) {
                    const uint2 d = __ldcs(reinterpret_cast<const uint2*>(p));
                    w[0] = d.x; w[1] = d.y;
                } else {
                    w[0] = __ldcs(reinterpret_cast<const uint32_t*>(p));
                }
                export_uyvy_split(w, &y, &uv);
                overlay_422_quad<E>(q, &y, &uv);
            } else {
                uv = export_422_quad<E>(f, q, &y);
            }
            export_uyvy_words(y, uv, w);
            if (full) __stcs(reinterpret_cast<uint2*>(p), make_uint2(w[0], w[1]));
            else __stcs(reinterpret_cast<uint32_t*>(p), w[0]);
        } else if (Fmt == GLAVA_B200_EXPORT_YUV422P) {
            uint8_t* const py = dst + (size_t) r * a.pitch + x;
            uint8_t* const pu = c.cb + (size_t) r * a.chroma_pitch + (x >> 1);
            uint8_t* const pv = c.cr + (size_t) r * a.chroma_pitch + (x >> 1);
            uint32_t y, u, v;
            if (native) {
                y = load_bytes(py, full ? 4 : 2); u = load_bytes(pu, full ? 2 : 1); v = load_bytes(pv, full ? 2 : 1);
                uint32_t uv = (u & 0xffu) | ((v & 0xffu) << 8) | ((u & 0xff00u) << 8) | ((v & 0xff00u) << 16);
                overlay_422_quad<E>(q, &y, &uv);
                u = export_cb_pair(uv); v = export_cr_pair(uv);
            } else {
                const uint32_t uv = export_422_quad<E>(f, q, &y);
                u = export_cb_pair(uv); v = export_cr_pair(uv);
            }
            store_bytes(py, y, full ? 4 : 2); store_bytes(pu, u, full ? 2 : 1); store_bytes(pv, v, full ? 2 : 1);
        } else {                                            // YUV422P10
            uint8_t* const py = dst + (size_t) r * a.pitch + 2 * (size_t) x;
            uint8_t* const pu = c.cb + (size_t) r * a.chroma_pitch + x;   // x / 2 samples of 2 bytes
            uint8_t* const pv = c.cr + (size_t) r * a.chroma_pitch + x;
            uint32_t y[2] = { 0u, 0u }, u, v;
            if (native) {
                if (full) {
                    const uint2 d = __ldcs(reinterpret_cast<const uint2*>(py));
                    y[0] = d.x; y[1] = d.y;
                    u = __ldcs(reinterpret_cast<const uint32_t*>(pu)); v = __ldcs(reinterpret_cast<const uint32_t*>(pv));
                } else {
                    y[0] = __ldcs(reinterpret_cast<const uint32_t*>(py));
                    u = __ldcs(reinterpret_cast<const unsigned short*>(pu)); v = __ldcs(reinterpret_cast<const unsigned short*>(pv));
                }
                overlay_422p10_quad<E>(q, y, &u, &v);
            } else {
                export_422p10_quad<E>(f, q, y, &u, &v);
            }
            if (full) {
                __stcs(reinterpret_cast<uint2*>(py), make_uint2(y[0], y[1]));
                __stcs(reinterpret_cast<uint32_t*>(pu), u); __stcs(reinterpret_cast<uint32_t*>(pv), v);
            } else {
                __stcs(reinterpret_cast<uint32_t*>(py), y[0]);
                __stcs(reinterpret_cast<unsigned short*>(pu), (unsigned short) u); __stcs(reinterpret_cast<unsigned short*>(pv), (unsigned short) v);
            }
        }
    }

    __device__ __forceinline__ void row(const OverlayPlanesEntry* e, uint8_t* dst, int r, int x, const uint32_t q[4]) const {
        if constexpr (k422) row422(true, dst, chroma(e), r, x, q);
        else row444(true, dst, chroma(e), r, x, q);
    }
    __device__ __forceinline__ void pair(uint8_t* dst, Chroma c, int j, int x, const uint32_t top[4], const uint32_t bot[4]) const {
        pair420(true, dst, c, j, x, top, bot);
    }
    __device__ __forceinline__ void item(const OverlayPlanesEntry* e, uint8_t* dst, int u, int x, const uint32_t top[4],
                                         const uint32_t bot[4], int y1) const {
        const Chroma c = chroma(e);
        if (k420) {
            pair420(a.native, dst, c, u, x, top, bot);
        } else if constexpr (k422) {
            row422(a.native, dst, c, 2 * u, x, top);
            if (y1 >= 0) row422(a.native, dst, c, 2 * u + 1, x, bot);
        } else {
            row444(a.native, dst, c, 2 * u, x, top);
            if (y1 >= 0) row444(a.native, dst, c, 2 * u + 1, x, bot);
        }
    }
};

template <typename Index, bool Band, int Fmt, int E>
__global__ void __launch_bounds__(256) overlay_planes_kernel(const __grid_constant__ OverlayPlanesArgs a) {
    overlay_walk<Index, Band>(OverlayPlanesBody<Fmt, E>(a));
}

template <int Fmt>
static void launch_planes_fade(const OverlayPlanesArgs& a, const ExportGrid& g, cudaStream_t st);   // DESIGN 4.20, below

template <int Fmt>
static void launch_planes(const OverlayPlanesArgs& a, const ExportGrid& g, cudaStream_t st) {
    if (a.fade) {
        launch_planes_fade<Fmt>(a, g, st);
        return;
    }
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.band) {
            if (g.narrow) overlay_planes_kernel<uint32_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_kernel<uint64_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        } else {
            if (g.narrow) overlay_planes_kernel<uint32_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_kernel<uint64_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        }
    });
}

template <int Fmt>
static void launch_planes_hdr(const OverlayPlanesArgs& a, const ExportGrid& g, cudaStream_t st);   // DESIGN 4.22, below

int launch_overlay_planes(const OverlayPlanesArgs& a, void* stream) {
    const int rows = a.band ? a.mark_rows : 2;
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) ((a.w + 127) >> 7) * (uint64_t) ((a.h + rows - 1) / rows));
    cudaStream_t st = (cudaStream_t) stream;
    if (a.enc >= GLB_ENC_PQ) {
        switch (a.format) {
        case GLAVA_B200_EXPORT_P010: launch_planes_hdr<GLAVA_B200_EXPORT_P010>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV420P10: launch_planes_hdr<GLAVA_B200_EXPORT_YUV420P10>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV444P10: launch_planes_hdr<GLAVA_B200_EXPORT_YUV444P10>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV422P10: launch_planes_hdr<GLAVA_B200_EXPORT_YUV422P10>(a, g, st); break;
        default: return fail(GLAVA_B200_EINVAL, "planes overlay launch: HDR on format %d", a.format);
        }
        return launch_status("planes overlay");
    }
    switch (a.format) {
    case GLAVA_B200_EXPORT_NV12: launch_planes<GLAVA_B200_EXPORT_NV12>(a, g, st); break;
    case GLAVA_B200_EXPORT_I420: launch_planes<GLAVA_B200_EXPORT_I420>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV444: launch_planes<GLAVA_B200_EXPORT_YUV444>(a, g, st); break;
    case GLAVA_B200_EXPORT_P010: launch_planes<GLAVA_B200_EXPORT_P010>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV420P10: launch_planes<GLAVA_B200_EXPORT_YUV420P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV444P10: launch_planes<GLAVA_B200_EXPORT_YUV444P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV422P: launch_planes<GLAVA_B200_EXPORT_YUV422P>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV422P10: launch_planes<GLAVA_B200_EXPORT_YUV422P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_UYVY: launch_planes<GLAVA_B200_EXPORT_UYVY>(a, g, st); break;
    default: return fail(GLAVA_B200_EINVAL, "planes overlay launch: format %d", a.format);
    }
    return launch_status("planes overlay");
}

// ---- overlay opacity (DESIGN 4.20) ----------------------------------------------------------------------------------------
// overlay_frames and overlay_planes at a per-entry opacity K (1..254 somewhere in the list; the host drops K = 0 entries and
// runs the plain kernels when every K is 255), K in the entry's pad word.  Every pixel is scaled by export_core.h fade_px
// (native opacity) or fade_opaque (any other: the stored colour with alpha 255) and then blended by the format's native
// item body, so a quad that is zero after scaling is neither loaded from the destination nor stored.  Items are
// overlay_walk's: bands under native opacity with marks, row pairs otherwise; under any other opacity no pixel is zero, so
// every row of the rectangle is read and written.

// overlay_walk's Body for overlay_frames' destinations (RGBA / BGRA rows, NV12 row pairs), the native blend only
template <int E>
struct OverlayFramesBody {
    const OverlayArgs& a;
    ExportFmt f;                                            // unused by the native blend: overlay_nv12 takes it
    bool bgra;
    __device__ __forceinline__ explicit OverlayFramesBody(const OverlayArgs& a_)
        : a(a_), f{ a_.format, 1, 0, 0u }, bgra(a_.format == GLAVA_B200_EXPORT_BGRA) {}
    static __device__ __forceinline__ uint8_t* dst(const ExportEntryUV* e) {
        return reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst)));
    }
    __device__ __forceinline__ bool pairs() const { return a.format == GLAVA_B200_EXPORT_NV12; }
    __device__ __forceinline__ uint8_t* chroma(const ExportEntryUV* e) const {
        return reinterpret_cast<uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&e->dst_uv)));
    }
    __device__ __forceinline__ void row(const ExportEntryUV*, uint8_t* dst, int r, int x, const uint32_t q[4]) const {
        overlay_rgba(dst + (size_t) r * a.pitch, x, a.w, bgra, q);
    }
    __device__ __forceinline__ void pair(uint8_t* dst, uint8_t* uv, int j, int x, const uint32_t top[4], const uint32_t bot[4]) const {
        overlay_nv12<E>(f, true, dst + (size_t) (2 * j) * a.pitch, uv + (size_t) j * a.pitch, a.pitch, x, a.w, top, bot);
    }
};

// overlay_walk's Body that scales every pixel by its entry's K and hands it to Inner's native row / pair
template <typename Args, typename Entry, typename Inner>
struct OverlayFadeBody {
    template <typename C> struct Faded { C c; uint32_t k; };
    const Args& a;
    Inner in;
    __device__ __forceinline__ explicit OverlayFadeBody(const Args& a_) : a(a_), in(a_) {}
    static __device__ __forceinline__ uint32_t k_of(const Entry* e) { return (uint32_t) __ldg(&e->pad); }
    static __device__ __forceinline__ uint8_t* dst(const Entry* e) { return Inner::dst(e); }
    __device__ __forceinline__ bool pairs() const { return in.pairs(); }
    __device__ __forceinline__ auto chroma(const Entry* e) const { return Faded<decltype(in.chroma(e))>{ in.chroma(e), k_of(e) }; }
    static __device__ __forceinline__ void scale(bool native, uint32_t k, const uint32_t q[4], uint32_t out[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = native ? fade_px(q[i], k) : fade_opaque(q[i], k);
    }
    // native, band items
    __device__ __forceinline__ void row(const Entry* e, uint8_t* dst, int r, int x, const uint32_t q[4]) const {
        uint32_t s[4];
        scale(true, k_of(e), q, s);
        in.row(e, dst, r, x, s);
    }
    template <typename C>
    __device__ __forceinline__ void pair(uint8_t* dst, const Faded<C>& c, int j, int x, const uint32_t top[4], const uint32_t bot[4]) const {
        uint32_t t[4], b[4];
        scale(true, c.k, top, t);
        scale(true, c.k, bot, b);
        in.pair(dst, c.c, j, x, t, b);
    }
    // row-pair items, any opacity
    __device__ __forceinline__ void item(const Entry* e, uint8_t* dst, int u, int x, const uint32_t top[4], const uint32_t bot[4],
                                         int y1) const {
        const uint32_t k = k_of(e);
        uint32_t t[4], b[4];
        scale(a.native, k, top, t);
        scale(a.native, k, bot, b);
        if (in.pairs()) {
            in.pair(dst, in.chroma(e), u, x, t, b);
        } else {
            in.row(e, dst, 2 * u, x, t);
            if (y1 >= 0) in.row(e, dst, 2 * u + 1, x, b);
        }
    }
};

template <typename Index, bool Band, int E>
__global__ void __launch_bounds__(256) overlay_fade_kernel(const __grid_constant__ OverlayArgs a) {
    overlay_walk<Index, Band>(OverlayFadeBody<OverlayArgs, ExportEntryUV, OverlayFramesBody<E>>(a));
}

template <typename Index, bool Band, int Fmt, int E>
__global__ void __launch_bounds__(256) overlay_planes_fade_kernel(const __grid_constant__ OverlayPlanesArgs a) {
    overlay_walk<Index, Band>(OverlayFadeBody<OverlayPlanesArgs, OverlayPlanesEntry, OverlayPlanesBody<Fmt, E>>(a));
}

static void launch_overlay_fade(const OverlayArgs& a, const ExportGrid& g, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.band) {
            if (g.narrow) overlay_fade_kernel<uint32_t, true, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_fade_kernel<uint64_t, true, E><<<g.blocks, 256, 0, st>>>(a);
        } else {
            if (g.narrow) overlay_fade_kernel<uint32_t, false, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_fade_kernel<uint64_t, false, E><<<g.blocks, 256, 0, st>>>(a);
        }
    });
}

template <int Fmt>
static void launch_planes_fade(const OverlayPlanesArgs& a, const ExportGrid& g, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.band) {
            if (g.narrow) overlay_planes_fade_kernel<uint32_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_fade_kernel<uint64_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        } else {
            if (g.narrow) overlay_planes_fade_kernel<uint32_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_fade_kernel<uint64_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        }
    });
}

// the 10-bit formats' plain and fade kernels under an HDR encoding (DESIGN 4.22)
template <int Fmt>
static void launch_planes_hdr(const OverlayPlanesArgs& a, const ExportGrid& g, cudaStream_t st) {
    for_hdr(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (a.fade) {
            if (a.band) {
                if (g.narrow) overlay_planes_fade_kernel<uint32_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
                else overlay_planes_fade_kernel<uint64_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            } else {
                if (g.narrow) overlay_planes_fade_kernel<uint32_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
                else overlay_planes_fade_kernel<uint64_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            }
        } else if (a.band) {
            if (g.narrow) overlay_planes_kernel<uint32_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_kernel<uint64_t, true, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        } else {
            if (g.narrow) overlay_planes_kernel<uint32_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
            else overlay_planes_kernel<uint64_t, false, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        }
    });
}

// ---- glava_b200_overlay_scaled (DESIGN 4.21) ---------------------------------------------------------------------------------
// The overlay of a downscaled, cropped frame.  Items are export_scaled_kernel's: (entry, output row — 4:2:0: row pair —, run
// of 32 output columns), one warp each, lane = output column, every pixel scaled_px's exact area average with its mark-aware
// footprint reads (native: of the stored pixels, zc 0; any other opacity: of the pixels made opaque, zc opaque black).  Each
// pixel is scaled by the entry's K through fade_px / fade_opaque (K = 255 is the identity, so there is no separate plain
// kernel), lanes past out_w hold zero, and the quad at X = 0 mod 4 is gathered by __shfl_down_sync into the lane that owns
// it, which runs the format's native body: overlay_rgba for RGBA / BGRA, OverlayPlanesBody's row / pair otherwise.  The
// bodies read the rectangle's width from their argument struct, so they get a view whose w is out_w.  An all-zero quad
// under native opacity is neither loaded from the picture nor stored.
template <typename Index, int Fmt, int E>
__global__ void __launch_bounds__(256) overlay_scaled_kernel(const __grid_constant__ OverlayScaledArgs a) {
    using Body = OverlayPlanesBody<Fmt, E>;
    constexpr bool rgba = Fmt == GLAVA_B200_EXPORT_RGBA;    // RGBA and BGRA (a.format says which)
    OverlayPlanesArgs view = {};                            // what the body reads: the rectangle's width and the pitches
    view.w = a.out_w; view.h = a.out_h; view.format = Fmt; view.native = 1;
    view.pitch = a.pitch; view.chroma_pitch = a.chroma_pitch;
    const Body body(view);
    const bool bgra = a.format == GLAVA_B200_EXPORT_BGRA;
    const ExportFmt f = { a.format, a.native ? 0 : 1, a.native, 0u };
    const ExportRecip rcp = { a.div_mul, a.div_shift };
    const uint32_t zc = a.native ? 0u : export_over(0u, 0u, 0);   // what a zero pixel becomes
    const Index runs = (Index) ((a.out_w + 31) >> 5), per = runs * (Index) (Body::k420 ? a.out_h >> 1 : a.out_h);
    const Index items = (Index) a.count * per;
    const Index warps = (Index) (((size_t) gridDim.x * blockDim.x) >> 5);
    const int lane = threadIdx.x & 31;
    for (Index it = (Index) (((size_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5); it < items; it += warps) {
        const Index k = it / per, rem = it - k * per;
        const int u = (int) (rem / runs), X = (int) (rem - (Index) u * runs) * 32 + lane;
        const bool active = X < a.out_w;
        const OverlayPlanesEntry* e = a.list + k;
        const int slot = __ldg(&e->slot);
        const uint32_t K = (uint32_t) __ldg(&e->pad);
        const uint32_t* frame = reinterpret_cast<const uint32_t*>(a.fb) + (size_t) slot * a.h * a.w;
        const ExportSpan sx = export_span(active ? X : 0, a.src_w, a.out_w);
        uint8_t* const dst = Body::dst(e);
        if constexpr (Body::k420) {
            uint32_t top = scaled_px<false>(a, f, frame, slot, 2 * u, active, sx, rcp, zc);
            uint32_t bot = scaled_px<false>(a, f, frame, slot, 2 * u + 1, active, sx, rcp, zc);
            top = !active ? 0u : a.native ? fade_px(top, K) : fade_opaque(top, K);
            bot = !active ? 0u : a.native ? fade_px(bot, K) : fade_opaque(bot, K);
            uint32_t t[4] = { top, 0u, 0u, 0u }, b[4] = { bot, 0u, 0u, 0u };
#pragma unroll
            for (int i = 1; i < 4; ++i) {
                t[i] = __shfl_down_sync(0xffffffffu, top, i);
                b[i] = __shfl_down_sync(0xffffffffu, bot, i);
            }
            if ((lane & 3) || !active) continue;
            body.pair(dst, body.chroma(e), u, X, t, b);
        } else {
            uint32_t px = scaled_px<false>(a, f, frame, slot, u, active, sx, rcp, zc);
            px = !active ? 0u : a.native ? fade_px(px, K) : fade_opaque(px, K);
            uint32_t q[4] = { px, 0u, 0u, 0u };
#pragma unroll
            for (int i = 1; i < 4; ++i) q[i] = __shfl_down_sync(0xffffffffu, px, i);
            if ((lane & 3) || !active) continue;
            if constexpr (rgba) overlay_rgba(dst + (size_t) u * a.pitch, X, a.out_w, bgra, q);
            else body.row(e, dst, u, X, q);
        }
    }
}

template <int Fmt>
static void launch_scaled_overlay(const OverlayScaledArgs& a, const ExportGrid& g, cudaStream_t st) {
    for_any_enc(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (g.narrow) overlay_scaled_kernel<uint32_t, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        else overlay_scaled_kernel<uint64_t, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
    });
}

// the 10-bit formats' kernels under an HDR encoding (DESIGN 4.22)
template <int Fmt>
static void launch_scaled_overlay_hdr(const OverlayScaledArgs& a, const ExportGrid& g, cudaStream_t st) {
    for_hdr(a.enc, [&](auto e) {
        constexpr int E = decltype(e)::value;
        if (g.narrow) overlay_scaled_kernel<uint32_t, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
        else overlay_scaled_kernel<uint64_t, Fmt, E><<<g.blocks, 256, 0, st>>>(a);
    });
}

int launch_overlay_scaled(const OverlayScaledArgs& a, void* stream) {
    const bool pairs = export_420(a.format);
    const ExportGrid g = export_grid((uint64_t) a.count * (uint64_t) ((a.out_w + 31) >> 5) *
                                     (uint64_t) (pairs ? a.out_h >> 1 : a.out_h));
    cudaStream_t st = (cudaStream_t) stream;
    if (a.enc >= GLB_ENC_PQ) {
        switch (a.format) {
        case GLAVA_B200_EXPORT_P010: launch_scaled_overlay_hdr<GLAVA_B200_EXPORT_P010>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV420P10: launch_scaled_overlay_hdr<GLAVA_B200_EXPORT_YUV420P10>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV444P10: launch_scaled_overlay_hdr<GLAVA_B200_EXPORT_YUV444P10>(a, g, st); break;
        case GLAVA_B200_EXPORT_YUV422P10: launch_scaled_overlay_hdr<GLAVA_B200_EXPORT_YUV422P10>(a, g, st); break;
        default: return fail(GLAVA_B200_EINVAL, "scaled overlay launch: HDR on format %d", a.format);
        }
        return launch_status("scaled overlay");
    }
    switch (a.format) {
    case GLAVA_B200_EXPORT_RGBA:
    case GLAVA_B200_EXPORT_BGRA:
        if (g.narrow) overlay_scaled_kernel<uint32_t, GLAVA_B200_EXPORT_RGBA, 0><<<g.blocks, 256, 0, st>>>(a);
        else overlay_scaled_kernel<uint64_t, GLAVA_B200_EXPORT_RGBA, 0><<<g.blocks, 256, 0, st>>>(a);
        break;
    case GLAVA_B200_EXPORT_NV12: launch_scaled_overlay<GLAVA_B200_EXPORT_NV12>(a, g, st); break;
    case GLAVA_B200_EXPORT_I420: launch_scaled_overlay<GLAVA_B200_EXPORT_I420>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV444: launch_scaled_overlay<GLAVA_B200_EXPORT_YUV444>(a, g, st); break;
    case GLAVA_B200_EXPORT_P010: launch_scaled_overlay<GLAVA_B200_EXPORT_P010>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV420P10: launch_scaled_overlay<GLAVA_B200_EXPORT_YUV420P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV444P10: launch_scaled_overlay<GLAVA_B200_EXPORT_YUV444P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV422P: launch_scaled_overlay<GLAVA_B200_EXPORT_YUV422P>(a, g, st); break;
    case GLAVA_B200_EXPORT_YUV422P10: launch_scaled_overlay<GLAVA_B200_EXPORT_YUV422P10>(a, g, st); break;
    case GLAVA_B200_EXPORT_UYVY: launch_scaled_overlay<GLAVA_B200_EXPORT_UYVY>(a, g, st); break;
    default: return fail(GLAVA_B200_EINVAL, "scaled overlay launch: format %d", a.format);
    }
    return launch_status("scaled overlay");
}

}  // namespace glb
