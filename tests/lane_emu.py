"""tests/emu/emu_lane.cu built with g++ and loaded once per process: lane_core.cuh run on the host (the lane engine's logic, lane by
lane) and the plain sequential slope-form scan the lane kernels must reproduce bit for bit (emu_slope_fibers_*).  One build shared by
the CPU emulation tests (test_lane_emulation.py) and the GPU tests of the lane kernels (test_gpu_lane.py)."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dp = C.POINTER(C.c_double)
fp = C.POINTER(C.c_float)


@functools.lru_cache(maxsize=None)
def _build():
    emu_dir = os.path.join(ROOT, "tests", "emu")
    so = os.path.join(emu_dir, "libptv_emu_lane.so")
    src = os.path.join(emu_dir, "emu_lane.cu")
    core = os.path.join(ROOT, "proxtv_b200", "csrc", "lane_core.cuh")
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in (src, core)):
        cuda_inc = "/usr/local/cuda/include"
        if not os.path.isdir(cuda_inc):
            return None
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + cuda_inc, "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", src, "-o", so])
    lib = C.CDLL(so)
    lib.emu_lane_f64.argtypes = [C.c_int, dp, dp, dp, dp, dp, C.c_longlong, C.c_int, C.c_longlong, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.POINTER(C.c_longlong)]
    lib.emu_lane_f32.argtypes = [C.c_int, fp, fp, fp, fp, fp, C.c_longlong, C.c_int, C.c_longlong, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.POINTER(C.c_longlong)]
    lib.emu_slope_seq_f64.argtypes = [dp, C.c_int, C.c_double, dp, C.POINTER(C.c_longlong)]
    lib.emu_slope_fibers_f64.argtypes = [dp, dp, C.c_longlong, C.c_int, C.c_longlong, C.c_double]
    lib.emu_slope_fibers_f32.argtypes = [fp, fp, C.c_longlong, C.c_int, C.c_longlong, C.c_float]
    lib.emu_plan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.emu_taskplan.argtypes = [C.c_int, C.c_longlong, C.c_longlong]; lib.emu_taskplan.restype = C.c_longlong
    return lib


def load():
    """The emulation library (built on first use, rebuilt when its sources are newer); skips the calling test without CUDA headers."""
    lib = _build()
    if lib is None:
        pytest.skip("CUDA headers not available")
    return lib


def slope_fibers(emu, a, nf, ln, inc, lam):
    """Sequential slope-form scan of every fiber of the (nf, ln, inc) slicing of the flat array `a` (float64 or float32; the float32
    form scans in double and rounds the results): the exact output of the lane engine's plain pass."""
    a = np.ascontiguousarray(a).ravel()
    out = np.full_like(a, np.nan)
    if a.dtype == np.float32:
        emu.emu_slope_fibers_f32(a.ctypes.data_as(fp), out.ctypes.data_as(fp), nf, ln, inc, np.float32(lam))
    else:
        emu.emu_slope_fibers_f64(a.ctypes.data_as(dp), out.ctypes.data_as(dp), nf, ln, inc, float(lam))
    return out
