"""The backward pass of DR2_TV on the host (DESIGN.md section 11), shared by test_dr2_vjp_cpu.py and test_gpu_dr2_vjp.py:

* ``forward`` -- DR2_TV with the lane engine's schedule (test_gpu_lane.py: dr_host, with separate column / row penalties), every prox
  pass the sequential slope-form scan the lane kernels reproduce bit for bit (lane_emu.slope_fibers), recording each pass output;
* ``backward`` -- the unrolled vector-Jacobian product of include/proxtv_b200.h (proxtv_DR2_TV_vjp_dev_*) restated in numpy: per pass
  vjp_emu.restate (segment means of the upstream gradient under that pass's segmentation), the combines in the storage type with the
  kernels' association, and the two order-dependent sums (start value term, penalty gradients) in float64;
* ``tape_bits`` -- the (F, U) segmentation tape of one pass output in numpy;
* ``load`` -- tests/emu/emu_vjp_tape.cu built with g++: the tape encoder and the tape-driven three passes of the backward kernels
  (proxtv_b200/csrc/vjp_core.cuh) on the CPU with a chosen chunk length.
Arrays are (B, M, N) images in C order (axis 0 of an image = M = the "columns" pass, axis 1 = N = the "rows" pass)."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

import vjp_emu
from lane_emu import slope_fibers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp = C.c_void_p
MAX_ITERS = 35


@functools.lru_cache(maxsize=None)
def _build():
    emu_dir = os.path.join(ROOT, "tests", "emu")
    so = os.path.join(emu_dir, "libptv_emu_vjp_tape.so")
    src = os.path.join(emu_dir, "emu_vjp_tape.cu")
    core = os.path.join(ROOT, "proxtv_b200", "csrc", "vjp_core.cuh")
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in (src, core)):
        cuda_inc = "/usr/local/cuda/include"
        if not os.path.isdir(cuda_inc):
            return None
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + cuda_inc, "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++", src, "-o", so])
    lib = C.CDLL(so)
    lib.emu_tape_f64.argtypes = [_vp, C.c_longlong, C.c_int, C.c_longlong, C.c_double, _vp, _vp, _vp]
    lib.emu_tape_f32.argtypes = [_vp, C.c_longlong, C.c_int, C.c_longlong, C.c_float, _vp, _vp, _vp]
    lib.emu_vjp_tape_f64.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_longlong, C.c_int, C.c_longlong, C.c_int]
    lib.emu_vjp_tape_f32.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_longlong, C.c_int, C.c_longlong, C.c_int]
    return lib


def load():
    """The emulation library (built on first use, rebuilt when its sources are newer); skips the calling test without CUDA headers."""
    lib = _build()
    if lib is None:
        pytest.skip("CUDA headers not available")
    return lib


def tape_words(n):
    """uint32 words of one bitset of an n-element tape: ceil(n / 32), padded to 256 bytes."""
    return ((n + 31) // 32 * 4 + 255) // 256 * 64


def tape_bits(y, nf, ln, inc, lam, W=None):
    """(F, U) bitsets (uint32 arrays of tape_words(nf * ln)) of the flat array y over the fibers (nf, ln, inc): bit i = element i and
    its successor i + inc -- (1, 0) fused (equal, weight > 0), (0, 1) successor greater, (0, 0) smaller or last sample, (1, 1) equal
    with a zero weight.  W: weights (nf, ln - 1) or None (penalty lam)."""
    y = np.ascontiguousarray(y).ravel()
    n = nf * ln
    idx = vjp_emu.flat_index(nf, ln, inc)                  # (nf, ln) positions
    a, b = y[idx[:, :-1]], y[idx[:, 1:]]
    wpos = (np.asarray(W) > 0) if W is not None else np.full(a.shape, lam > 0)
    f = np.zeros(n, dtype=bool)
    u = np.zeros(n, dtype=bool)
    f[idx[:, :-1]] = a == b
    u[idx[:, :-1]] = (b > a) | ((a == b) & ~wpos)
    nw = tape_words(n)
    out = []
    for bits in (f, u):
        full = np.zeros(nw * 32, dtype=np.uint64)
        full[:n] = bits
        out.append((full.reshape(nw, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32))
    return out[0], out[1]


def emulate_tape(emu, F, U, G, nf, ln, inc, chunk=0, want_gw=True):
    """The device's tape-driven three passes on the host; G (nf, ln) in the fibers' order; returns gx (nf, ln), gw (nf, ln-1)."""
    T = G.dtype
    g = vjp_emu.to_flat(G, inc)
    gx = np.full(nf * ln, np.nan, dtype=T)
    gw = np.full(nf * max(ln - 1, 0), np.nan, dtype=T) if want_gw else None
    fn = emu.emu_vjp_tape_f32 if T == np.float32 else emu.emu_vjp_tape_f64
    fn(F.ctypes.data, U.ctypes.data, g.ctypes.data, gx.ctypes.data, gw.ctypes.data if gw is not None else None, nf, ln, inc, chunk)
    return vjp_emu.from_flat(gx, nf, ln, inc), (vjp_emu.from_flat(gw, nf, ln - 1, inc) if gw is not None else None)


# ---------------------------------------------------------------------------------------------------------------- the schedule
def _cols(emu, a, lam):
    B, M, N = a.shape
    return slope_fibers(emu, np.ascontiguousarray(a.transpose(0, 2, 1)), B * N, M, 1, lam).reshape(B, N, M).transpose(0, 2, 1)


def _rows(emu, a, lam):
    B, M, N = a.shape
    return slope_fibers(emu, np.ascontiguousarray(a), B * M, N, 1, lam).reshape(B, M, N)


def forward(emu, Y, w1, w2, maxit=0):
    """DR2_TV of every image of Y (B, M, N) on the lane schedule; returns (out, passes) with passes the 2K + 1 recorded pass outputs
    in execution order (p = 0: row pass of k = 0; p = 2k - 1 / 2k: column / row pass of iteration k; the last two: the final pair).
    Arithmetic in the storage type; the start value is the float64 sum, doubled, divided by M N, rounded to the storage type."""
    T = Y.dtype.type
    B, M, N = Y.shape
    K = MAX_ITERS if maxit <= 0 else maxit
    mean2 = (2.0 * Y.astype(np.float64).reshape(B, -1).sum(axis=1)) / float(M * N)
    t = np.ascontiguousarray(np.broadcast_to(mean2.astype(T)[:, None, None], Y.shape))
    w1, w2 = T(w1), T(w2)
    passes = []
    for k in range(K + 1):
        if k == 0:
            x1 = t.copy()
        else:
            x1 = _cols(emu, t, w1)
            passes.append(x1)
        d = t - x1
        if k == K:
            out = _rows(emu, Y - d, w2)
            passes.append(out)
            return out, passes
        x2 = _rows(emu, Y - (T(2) * d - t), w2)
        passes.append(x2)
        t = d + x2


def _S(X, G, lam, col):
    """Segment means of G under the segmentation of the pass output X (B, M, N) along axis 0 (col) or 1, and the per-image sums of
    its edge gradients gw (float64)."""
    B, M, N = X.shape
    if col:
        f = lambda a: np.ascontiguousarray(a.transpose(0, 2, 1)).reshape(B * N, M)          # noqa: E731
        gx, gw = vjp_emu.restate(f(X), f(G), lam)
        gx = gx.reshape(B, N, M).transpose(0, 2, 1)
    else:
        gx, gw = vjp_emu.restate(X.reshape(B * M, N), G.reshape(B * M, N), lam)
        gx = gx.reshape(B, M, N)
    return np.ascontiguousarray(gx), gw.astype(np.float64).reshape(B, -1).sum(axis=1)


def backward(passes, G, w1, w2, maxit=0):
    """gY (like G, storage type) and glam (B, 2) float64 -- [d/dw1, d/dw2] per image -- for the upstream gradient G of forward()'s
    output; the recurrence of proxtv_b200/csrc/dr2_vjp.cu with the same associations."""
    T = G.dtype.type
    B, M, N = G.shape
    K = MAX_ITERS if maxit <= 0 else maxit
    w1, w2 = T(w1), T(w2)
    glam = np.zeros((B, 2))
    a, s = _S(passes[2 * K], G, w2, False); glam[:, 1] += s
    sc, s = _S(passes[2 * K - 1], a, w1, True); glam[:, 0] += s
    gY = a.copy()
    g = sc - a
    for k in range(K - 1, -1, -1):
        a, s = _S(passes[2 * k], g, w2, False); glam[:, 1] += s
        gY = gY + a
        h = g - T(2) * a
        if k > 0:
            sc, s = _S(passes[2 * k - 1], h, w1, True); glam[:, 0] -= s
        else:                                               # the prox of the constant start image
            sc, _ = _S(np.zeros_like(h), h, T(1) if w1 > 0 else T(0), True)
        g = (a + h) - sc
    sums = g.astype(np.float64).reshape(B, -1).sum(axis=1)
    gY = (gY.astype(np.float64) + ((2.0 * sums) / float(M * N))[:, None, None]).astype(T)
    return gY, glam
