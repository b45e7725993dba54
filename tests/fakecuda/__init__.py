"""TEST INFRASTRUCTURE — the library's host code (capi.cu, config.cpp) built with g++ against a fake CUDA runtime and fake
kernel launchers (fakecuda.cpp), for testing resource ownership and the rebuild path without a GPU."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "glava_b200", "csrc")
BUF, PINNED, EVENT, STREAM = range(4)
_lib = None


def cuda_include():
    """the toolkit's include directory (cuda_runtime.h declares the runtime fakecuda.cpp defines), or None"""
    nvcc = shutil.which("nvcc")
    roots = [os.environ.get("CUDA_HOME"), os.path.dirname(os.path.dirname(nvcc)) if nvcc else None, "/usr/local/cuda"]
    for root in roots:
        if root and os.path.exists(os.path.join(root, "include", "cuda_runtime.h")):
            return os.path.join(root, "include")
    return None


def lib():
    global _lib
    if _lib is None:
        out = tempfile.mkdtemp(prefix="glava_fakecuda_")
        so = os.path.join(out, "libglava_fakecuda.so")
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas",
                        "-I", cuda_include(), "-x", "c++", "-include", "cuda_runtime.h", "-o", so,
                        os.path.join(CSRC, "capi.cu"), os.path.join(CSRC, "config.cpp"), os.path.join(HERE, "fakecuda.cpp"),
                        "-lpthread", "-Wl,-Bsymbolic"], check=True)
        L = C.CDLL(so)
        shutil.rmtree(out)                                            # stays mapped
        L.fake_first_violation.restype = C.c_char_p
        L.fake_trace.restype = C.c_char_p
        for f in ("fake_creations", "fake_live", "fake_launches", "fake_violations", "fake_stale", "fake_reached"):
            getattr(L, f).restype = C.c_long
        L.fake_fail_at.argtypes = [C.c_long]
        L.fake_live.argtypes = [C.c_int]
        _lib = L
    return _lib


def live(L):
    """live (buffers, pinned buffers, events, streams)"""
    return tuple(L.fake_live(k) for k in (BUF, PINNED, EVENT, STREAM))
