"""TEST INFRASTRUCTURE — capi.cu, export.cpp and config.cpp built with g++ against tests/fakecuda's runtime and launchers,
plus what the caller-buffer exports add: cudaPointerGetAttributes (device memory = the byte ranges the test registers) and
the three export launchers, which count their calls, record their last arguments and refuse what the kernels could not
run.  One build serves test_export_core.py, test_export_scaled_core.py and test_overlay_core.py."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

from tests import fakecuda

STUBS = r"""
#include "internal.h"
#include <map>
static std::map<uintptr_t, size_t> g_dev;                 // device allocations: start -> bytes
static long g_launches = 0;
static glb::ScaledArgs g_scaled;
static glb::OverlayArgs g_overlay;
extern "C" void export_fake_device(const void* p, size_t n) { g_dev[(uintptr_t) p] = n; }
extern "C" void export_fake_forget(const void* p) { g_dev.erase((uintptr_t) p); }
extern "C" long export_fake_launches(void) { return g_launches; }
extern "C" void export_fake_last(int* out) {
    out[0] = g_scaled.src_x; out[1] = g_scaled.src_y; out[2] = g_scaled.src_w; out[3] = g_scaled.src_h; out[4] = g_scaled.out_w;
    out[5] = g_scaled.out_h; out[6] = g_scaled.count; out[7] = g_scaled.over;
}
extern "C" void overlay_fake_last(int* out) { out[0] = g_overlay.count; out[1] = g_overlay.band; out[2] = g_overlay.native; out[3] = g_overlay.format; }
extern "C" cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p) {
    *a = cudaPointerAttributes();
    auto it = g_dev.upper_bound((uintptr_t) p);            // a pointer anywhere inside an allocation
    const bool dev = it != g_dev.begin() && (uintptr_t) p < std::prev(it)->first + std::prev(it)->second;
    a->type = dev ? cudaMemoryTypeDevice : cudaMemoryTypeUnregistered;
    a->device = 0;
    return cudaSuccess;
}
// overlay_geometry_check on plain addresses: NV12 (chroma rows at uv[i]) when uv is non-null
extern "C" int t_geometry(int w, int h, int count, const uintptr_t* dst, const uintptr_t* uv, size_t pitch, uintptr_t fb, size_t fb_bytes) {
    glava_b200_export d = {};
    d.format = uv ? GLAVA_B200_EXPORT_NV12 : GLAVA_B200_EXPORT_RGBA;
    d.pitch = pitch;
    const uint8_t* f = (const uint8_t*) fb;
    return glb::overlay_geometry_check(w, h, count, (void* const*) dst, (void* const*) uv, d, &f, &fb_bytes, 1, "t_geometry");
}
namespace glb {
int launch_export(const ExportArgs& a, void*) {
    ++g_launches;
    return a.fb && a.list && a.count > 0 && (!a.marks || a.mark_rows > 0) ? 0 : fail(GLAVA_B200_EINVAL, "export launch: missing buffers");
}
int launch_export_scaled(const ScaledArgs& a, void*) {
    ++g_launches; g_scaled = a;
    return a.fb && a.list && a.count > 0 && (!a.marks || a.mark_rows > 0) ? 0 : fail(GLAVA_B200_EINVAL, "scaled launch: missing buffers");
}
int launch_overlay(const OverlayArgs& a, void*) {
    ++g_launches; g_overlay = a;
    return a.fb && a.list && a.count > 0 && (!a.band || (a.marks && a.mark_rows > 0 && a.native)) ? 0
                                                                                                : fail(GLAVA_B200_EINVAL, "overlay launch: bad arguments");
}
}
"""
_lib = None


def lib():
    """the library, built on first use (None without the toolkit's headers); L.renderer(module, batch, **params) makes a
    handle, L.device_buf(nbytes) a registered device buffer, and L.cudaFree unregisters what it frees (the host allocator
    may hand those bytes out again)"""
    global _lib
    inc = fakecuda.cuda_include()
    if _lib is not None or inc is None:
        return _lib
    from glava_b200.api import Export, ExportScale, Params
    out = tempfile.mkdtemp(prefix="glava_export_fake_")
    src, so = os.path.join(out, "export_fake.cpp"), os.path.join(out, "libexport_fake.so")
    with open(src, "w") as f:
        f.write(STUBS)
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-I", inc,
                    "-I", fakecuda.CSRC, "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                    os.path.join(fakecuda.CSRC, "capi.cu"), os.path.join(fakecuda.CSRC, "export.cpp"),
                    os.path.join(fakecuda.CSRC, "config.cpp"), os.path.join(fakecuda.HERE, "fakecuda.cpp"), src, "-lpthread",
                    "-Wl,-Bsymbolic"], check=True)
    L = C.CDLL(so)
    shutil.rmtree(out)                                                # stays mapped
    vp, i32, P, E, S = C.c_void_p, C.c_int, C.POINTER(Params), C.POINTER(Export), C.POINTER(ExportScale)
    sig = {
        "glava_b200_default_params": (i32, [P, C.c_char_p]), "glava_b200_new": (vp, [P, i32, i32]),
        "glava_b200_destroy": (None, [vp]), "glava_b200_reconfigure": (i32, [vp, P]), "glava_b200_get_params": (i32, [vp, P]),
        "glava_b200_update": (i32, [vp, vp, vp, C.c_size_t, i32]), "glava_b200_last_error": (C.c_char_p, []),
        "glava_b200_set_abort_hook": (None, [vp]), "glava_b200_framebuffer_device": (vp, [vp]),
        "glava_b200_export_frames": (i32, [vp, vp, i32, vp, E, vp, vp]),
        "glava_b200_export_bytes": (i32, [vp, E, C.POINTER(C.c_size_t)]),
        "glava_b200_export_scaled": (i32, [vp, vp, i32, vp, vp, E, S, vp, vp]),
        "glava_b200_export_scaled_bytes": (i32, [vp, E, S, C.POINTER(C.c_size_t)]),
        "glava_b200_overlay_frames": (i32, [vp, vp, i32, vp, vp, E, vp, vp]),
        "cudaMalloc": (i32, [C.POINTER(vp), C.c_size_t]), "cudaFree": (i32, [vp]), "cudaEventCreate": (i32, [C.POINTER(vp)]),
        "cudaEventDestroy": (i32, [vp]), "fake_trace": (C.c_char_p, []), "fake_fail_at": (None, [C.c_long]),
        "fake_live": (C.c_long, [i32]), "export_fake_device": (None, [vp, C.c_size_t]), "export_fake_forget": (None, [vp]),
        "export_fake_launches": (C.c_long, []), "export_fake_last": (None, [vp]), "overlay_fake_last": (None, [vp]),
        "t_geometry": (i32, [i32, i32, i32, vp, vp, C.c_size_t, C.c_size_t, C.c_size_t]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    L._quiet = C.CFUNCTYPE(None, C.c_char_p)(lambda msg: None)
    L.glava_b200_set_abort_hook(C.cast(L._quiet, vp))

    def renderer(module="bars", batch=2, **kw):
        p = Params()
        assert L.glava_b200_default_params(C.byref(p), module.encode()) == 0
        for k, v in kw.items():
            setattr(p, k, v)
        h = L.glava_b200_new(C.byref(p), batch, 0)
        assert h, L.glava_b200_last_error()
        return C.c_void_p(h), p

    def device_buf(nbytes=1 << 16):
        b = C.c_void_p()
        assert L.cudaMalloc(C.byref(b), nbytes) == 0
        L.export_fake_device(b, nbytes)
        return b

    free = L.cudaFree

    def cuda_free(p):
        L.export_fake_forget(p)
        return free(p)

    L.renderer, L.device_buf, L.cudaFree = renderer, device_buf, cuda_free
    _lib = L
    return _lib


def desc_of(fmt, pitch, flags=0, uv=0):
    from glava_b200.api import Export
    d = Export()
    d.format, d.flags, d.pitch, d.uv_offset = fmt, flags, pitch, uv
    return d
