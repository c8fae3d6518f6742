"""The backward pass of the batched 1D prox on the host, twice over:

* ``restate`` -- the contract of include/proxtv_b200.h (proxtv_prox_fibers_vjp_dev_*) restated in numpy: THE pin.  Every segment's sum
  runs left to right from 0.0 in float64 (numpy's ``cumsum`` and elementwise ``+`` are sequential, unlike ``sum``);
* ``load`` -- tests/emu/emu_vjp.cu built with g++: proxtv_b200/csrc/vjp_core.cuh (the device kernels' chunk scan, carry and fix-up) run
  on the CPU with a chosen chunk length, so the CPU suite can check that the work split changes no bit.
Shared by test_vjp_cpu.py and test_gpu_vjp.py."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p


@functools.lru_cache(maxsize=None)
def _build():
    emu_dir = os.path.join(ROOT, "tests", "emu")
    so = os.path.join(emu_dir, "libptv_emu_vjp.so")
    src = os.path.join(emu_dir, "emu_vjp.cu")
    core = os.path.join(ROOT, "proxtv_b200", "csrc", "vjp_core.cuh")
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in (src, core)):
        cuda_inc = "/usr/local/cuda/include"
        if not os.path.isdir(cuda_inc):
            return None
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + cuda_inc, "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", src, "-o", so])
    lib = C.CDLL(so)
    lib.emu_vjp_f64.argtypes = [_vp, _vp, _vp, _vp, C.c_longlong, C.c_int, C.c_longlong, C.c_double, _vp, C.c_int]
    lib.emu_vjp_f32.argtypes = [_vp, _vp, _vp, _vp, C.c_longlong, C.c_int, C.c_longlong, C.c_float, _vp, C.c_int]
    return lib


def load():
    """The emulation library (built on first use, rebuilt when its sources are newer); skips the calling test without CUDA headers."""
    lib = _build()
    if lib is None:
        pytest.skip("CUDA headers not available")
    return lib


def flat_index(nf, ln, inc):
    """(nf, ln) positions of the fibers' samples in a flat array under the slicing rule (nf, ln, inc) (nf a multiple of inc)."""
    f = np.arange(nf)[:, None]
    return (f // inc) * inc * ln + f % inc + np.arange(ln)[None, :] * inc


def to_flat(F, inc):
    nf, ln = F.shape
    out = np.empty(nf * ln, dtype=F.dtype)
    out[flat_index(nf, ln, inc)] = F
    return out


def from_flat(v, nf, ln, inc):
    return np.asarray(v)[flat_index(nf, ln, inc)]


def restate(Y, G, lam, W=None):
    """gx (nf, len) and gw (nf, len-1) of the contract for forward outputs Y and upstream gradients G (nf, len), float64 or float32,
    penalty lam or per-edge weights W (nf, len-1); results in the storage type."""
    T = Y.dtype
    nf, ln = Y.shape
    if nf == 0 or ln == 0:
        return np.zeros((nf, ln), T), np.zeros((nf, max(ln - 1, 0)), T)
    wpos = (W > 0) if W is not None else np.full((nf, ln - 1), lam > 0)
    fused = (Y[:, 1:] == Y[:, :-1]) & wpos
    start = np.ones((nf, ln), dtype=bool)
    start[:, 1:] = ~fused
    a = np.flatnonzero(start.ravel())
    cnt = np.diff(np.append(a, nf * ln))
    g = G.astype(np.float64).ravel()
    s = np.zeros(a.size)
    short = np.flatnonzero(cnt <= 64)
    for k in range(int(cnt[short].max()) if short.size else 0):     # position k of every short segment at once, in order
        sel = short[cnt[short] > k]
        s[sel] = s[sel] + g[a[sel] + k]
    for j in np.flatnonzero(cnt > 64):
        s[j] = np.cumsum(np.concatenate(([0.0], g[a[j]:a[j] + cnt[j]])))[-1]
    mt = (s / cnt.astype(np.float64)).astype(T)
    gx = np.repeat(mt, cnt).reshape(nf, ln)
    gxd = gx.astype(np.float64)
    sg = np.sign(Y[:, 1:].astype(np.float64) - Y[:, :-1].astype(np.float64))
    gw = np.where(fused, 0.0, sg * (gxd[:, :-1] - gxd[:, 1:])).astype(T)
    return gx, gw


def emulate(emu, Y, G, lam, W=None, chunk=0, inc=1, want_gw=True):
    """The device's three passes on the host with chunk length `chunk` (0: whole fibers), over the fibers laid out with stride inc."""
    T = Y.dtype
    nf, ln = Y.shape
    y, g = to_flat(Y, inc), to_flat(G, inc)
    gx = np.full(nf * ln, np.nan, dtype=T)
    gw = np.full(nf * max(ln - 1, 0), np.nan, dtype=T) if want_gw else None
    w = to_flat(np.ascontiguousarray(W, dtype=T), inc) if W is not None else None
    fn = emu.emu_vjp_f32 if T == np.float32 else emu.emu_vjp_f64
    fn(y.ctypes.data, g.ctypes.data, gx.ctypes.data, gw.ctypes.data if gw is not None else None, nf, ln, inc,
       T.type(lam), w.ctypes.data if w is not None else None, chunk)
    return from_flat(gx, nf, ln, inc), (from_flat(gw, nf, ln - 1, inc) if gw is not None else None)
