"""CPU test of the lane engine with one penalty per lane (per-fiber penalties, DESIGN.md section 16.1): tests/emu/emu_lane_lamf.cu runs
lane_core.cuh -- the code the LAMF instantiation of the lane kernel executes -- on the host, each lane scanning, finishing and being
repaired with its own fiber's penalty lamf[j / fpi].  Every fiber must equal the plain sequential slope-form scan of that fiber with its
own penalty (emu_slope_fibers_*) bit for bit: groups that split a warp (fpi not a multiple of 32), both layouts (contiguous fibers
drained in boxes, strided fibers drained by rows), float64 and float32, whole fibers and forced chunking, with and without halo (halo 0:
every chunk boundary goes through the repair path).  No GPU needed."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

from lane_emu import load as load_lane_emu
from lane_emu import slope_fibers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def _build():
    emu_dir = os.path.join(ROOT, "tests", "emu")
    so = os.path.join(emu_dir, "libptv_emu_lane_lamf.so")
    srcs = [os.path.join(emu_dir, f) for f in ("emu_lane_lamf.cu", "emu_lane.cu")] + [os.path.join(ROOT, "proxtv_b200", "csrc", "lane_core.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in srcs):
        cuda_inc = "/usr/local/cuda/include"
        if not os.path.isdir(cuda_inc):
            return None
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + cuda_inc, "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", srcs[0], "-o", so])
    lib = C.CDLL(so)
    for t, sfx in ((C.c_double, "f64"), (C.c_float, "f32")):
        p = C.POINTER(t)
        getattr(lib, "emu_lane_lamf_" + sfx).argtypes = [p, p, C.c_longlong, C.c_int, C.c_longlong, p, C.c_longlong, C.c_int, C.c_int,
                                                         C.POINTER(C.c_longlong)]
    return lib


@pytest.fixture(scope="module")
def emu():
    lib = _build()
    if lib is None:
        pytest.skip("CUDA headers not available")
    return lib


def lane_lamf(lib, A, nf, ln, inc, lamf, fpi, clen, halo):
    t = C.c_float if A.dtype == np.float32 else C.c_double
    X = np.full_like(A, np.nan)
    st = (C.c_longlong * 8)()
    f = lib.emu_lane_lamf_f32 if A.dtype == np.float32 else lib.emu_lane_lamf_f64
    f(A.ctypes.data_as(C.POINTER(t)), X.ctypes.data_as(C.POINTER(t)), nf, ln, inc, lamf.ctypes.data_as(C.POINTER(t)), fpi, clen, halo, st)
    return X, st[5]


def test_per_lane_penalty_is_the_sequential_scan_per_fiber(emu):
    seq = load_lane_emu()
    rng = np.random.default_rng(5)
    ln = 300
    values = np.array([0.05, 0.2, 1.0, 5.0, 1e-12, 50.0, 0.5])
    repairs = 0
    for dt in (np.float64, np.float32):
        for fpi in (1, 7, 32, 33):
            nf = 4 * 33 * (8 if fpi == 1 else 1)                 # partial last fiber groups; 7 and 33 split warps between two items
            nf -= nf % fpi
            blocks = np.repeat(rng.normal(0, 1, (nf, ln // 16 + 1)), 16, axis=1)[:, :ln] + rng.normal(0, 0.3, (nf, ln))
            lamf = values[np.arange(nf // fpi) % len(values)].astype(dt)
            for inc in (nf, 1):                                  # strided fibers (one slab), contiguous fibers
                A = np.ascontiguousarray((blocks.T if inc > 1 else blocks).astype(dt)).ravel()
                want = np.full_like(A, np.nan)
                idx = (np.arange(nf * ln).reshape(ln, nf).T if inc > 1 else np.arange(nf * ln).reshape(nf, ln))
                for v in np.unique(lamf):
                    sel = idx[lamf[np.arange(nf) // fpi] == v].ravel()
                    want[sel] = slope_fibers(seq, A, nf, ln, inc, v)[sel]
                for clen, halo in ((0, 32), (64, 32), (48, 0)):
                    X, rep = lane_lamf(emu, A, nf, ln, inc, lamf, fpi, clen, halo)
                    assert np.array_equal(X, want), (dt.__name__, fpi, inc, clen, halo)
                    if clen and halo == 0:
                        assert rep >= nf
                    repairs += rep
    assert repairs > 1000
