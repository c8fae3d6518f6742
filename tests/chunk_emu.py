"""Host emulations of the taut-string routes of the batched 1D prox, built with nvcc (host code only, -fmad=false, -ffp-contract=off)
and loaded once per process:

* seq()     -- tests/emu/emu_seq.cu: the sequential kernel's scan, Scan<T> of taut_scan.cuh driven fiber by fiber in T arithmetic
               (emu_seq_fibers_*);
* chunked() -- tests/emu/emu_chunked.cu: the chunked kernel's per-lane phases run lane by lane (emu_chunked_*).

Used by the CPU tests of test_seq_emulation.py and the GPU tests of the 1D prox's dispatch routes (test_gpu_prox1d_routes.py).  Each
library is compiled to a private file name and moved into place in one step, so processes that build it at the same time never see or
overwrite a partly written library."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "emu")
CORE = [os.path.join(ROOT, "proxtv_b200", "csrc", f) for f in ("chunk_core.cuh", "taut_scan.cuh")]
dp = C.POINTER(C.c_double)
fp = C.POINTER(C.c_float)


def _compile(src, so):
    """Build `src` into `so` unless `so` is newer than the sources; None without nvcc."""
    src = os.path.join(EMU_DIR, src)
    so = os.path.join(EMU_DIR, so)
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in [src] + CORE):
        nvcc = "/usr/local/cuda/bin/nvcc"
        if not os.path.exists(nvcc):
            return None
        tmp = "%s.%d.tmp" % (so, os.getpid())
        subprocess.check_call([nvcc, "-O2", "-std=c++17", "-arch=sm_90a", "-fmad=false", "--expt-relaxed-constexpr",
                               "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-x", "cu", src, "-o", tmp])
        os.replace(tmp, so)
    return C.CDLL(so)


@functools.lru_cache(maxsize=None)
def _seq():
    lib = _compile("emu_seq.cu", "libptv_emu_seq.so")
    if lib is not None:
        lib.emu_seq_fibers_f64.argtypes = [dp, dp, C.c_longlong, C.c_int, C.c_longlong, C.c_double, dp]
        lib.emu_seq_fibers_f32.argtypes = [fp, fp, C.c_longlong, C.c_int, C.c_longlong, C.c_float, fp]
        lib.emu_seq_fibers_f64.restype = lib.emu_seq_fibers_f32.restype = None
    return lib


@functools.lru_cache(maxsize=None)
def _chunked():
    lib = _compile("emu_chunked.cu", "libptv_emu_chunked.so")
    if lib is not None:
        lib.emu_chunked_f32.argtypes = [fp, C.c_int, C.c_float, fp, fp, C.c_int, C.POINTER(C.c_int)]
    return lib


def _need(lib):
    if lib is None:
        pytest.skip("nvcc not available")
    return lib


def seq_fibers(a, nf, ln, inc, lam, w=None):
    """The sequential kernel's result for every fiber of the (nf, ln, inc) slicing of the flat array `a`, in a's storage type (float64 or
    float32 arithmetic); w: per-edge weights laid out like the fibers with ln - 1 samples each, or None for the uniform penalty lam.
    Elements that belong to no fiber are NaN."""
    lib = _need(_seq())
    a = np.ascontiguousarray(a).ravel()
    out = np.full_like(a, np.nan)
    f32 = a.dtype == np.float32
    ptr_t, fn = (fp, lib.emu_seq_fibers_f32) if f32 else (dp, lib.emu_seq_fibers_f64)
    wp = None
    if w is not None:
        w = np.ascontiguousarray(w, dtype=a.dtype).ravel()
        wp = w.ctypes.data_as(ptr_t)
    fn(a.ctypes.data_as(ptr_t), out.ctypes.data_as(ptr_t), nf, ln, inc, np.float32(lam) if f32 else float(lam), wp)
    return out


def chunked_f32(y, lam, w=None):
    """One float32 fiber through the emulated chunked CTA (32-sample chunks)."""
    lib = _need(_chunked())
    y = np.ascontiguousarray(y, dtype=np.float32); x = np.empty_like(y); r = C.c_int(0)
    wp = None
    if w is not None:
        w = np.ascontiguousarray(w, dtype=np.float32); wp = w.ctypes.data_as(fp)
    rc = lib.emu_chunked_f32(y.ctypes.data_as(fp), y.size, np.float32(lam), wp, x.ctypes.data_as(fp), 0, C.byref(r))
    assert rc == 0, "emulated CTA broke the barrier discipline (rc=%d)" % rc
    return x
