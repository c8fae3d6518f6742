"""GPU tests of the weighted Condat / Chambolle-Pock 2D TV-L1 prox (proxtv_CP2W_TV_*, cp2.cu, DESIGN.md section 15.1): float64 bit for
bit equal to the weighted port (tests/cp2w_port.c, pinned by tests/test_cp2w_cpu.py), iteration counts included, through the host
batched entry point in both storage orders and torch tensors of both memory orders; constant maps equal the unweighted solver; mixed
batches; float32 close to the port; the device entry point on a stream; the refusal of gradients."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import relerr
from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cp2w_port as port  # noqa: E402

pytestmark = pytest.mark.gpu
METHODS = {0: "condat", 1: "chambolle-pock"}
SHAPES = [(1, 1), (1, 9), (9, 1), (2, 2), (2, 7), (7, 2), (33, 47), (64, 64), (128, 96)]


def maps(kind, M, N, seed):
    """(w_col (M-1, N), w_row (M, N-1)): 'random' -- the two axes from different ranges; 'zeros' -- random with about a third of the
    edges exactly 0; 'const' -- 0.2 everywhere."""
    rng = np.random.default_rng(seed)
    if kind == "const":
        return np.full((M - 1, N), 0.2), np.full((M, N - 1), 0.2)
    w1 = rng.uniform(0.05, 0.6, (M - 1, N)); w2 = rng.uniform(0.0, 0.15, (M, N - 1))
    if kind == "zeros":
        w1[rng.random(w1.shape) < 0.33] = 0.0; w2[rng.random(w2.shape) < 0.33] = 0.0
    return w1, w2


def host_batched(ptv, Y, W1, W2, alg, maxit, row_major):
    """proxtv_CP2W_TV_batched_f64 on one image in the given storage order: (X as an (M, N) array, info)."""
    M, N = Y.shape
    order = "C" if row_major else "F"
    y = np.require(Y, np.float64, [order]); w1 = np.require(W1, np.float64, [order]); w2 = np.require(W2, np.float64, [order])
    x = np.zeros((M, N), order=order); info = np.zeros(3)
    ok = ptv.load().proxtv_CP2W_TV_batched_f64(M, N, 1, row_major, y.ctypes.data, w1.ctypes.data, w2.ctypes.data, x.ctypes.data, alg,
                                                int(maxit), info.ctypes.data)
    assert ok == 1 and info[2] == 0, ptv._lib.last_error()
    return x, info


def test_bitwise_against_port(ptv):
    import torch
    k = 0
    for M, N in SHAPES:
        Y = O.gen_cfg2(M, N, seed=40 + k, block=4)
        for kind in ("random", "zeros", "const"):
            W1, W2 = maps(kind, M, N, seed=k)
            k += 1
            for alg, m in METHODS.items():
                for maxit in (1, 7, 0):
                    want, winfo = port.cp2w_tv(Y, W1, W2, alg, maxit)
                    case = (M, N, kind, m, maxit)
                    for rm in (0, 1):
                        got, ginfo = host_batched(ptv, Y, W1, W2, alg, maxit, rm)
                        assert np.array_equal(got, want), case + (rm,)
                        assert ginfo[0] == winfo[0], case + (rm, ginfo[0], winfo[0])
                    rmt = torch.tensor(np.ascontiguousarray(Y), device="cuda")                 # C order: row_major = 1
                    cmt = torch.tensor(np.ascontiguousarray(Y.T), device="cuda").t()          # column-major: row_major = 0
                    w1t, w2t = torch.tensor(W1, device="cuda"), torch.tensor(W2, device="cuda")
                    a = ptv.tv1w_2d(rmt, w1t, w2t, max_iters=maxit, method=m)
                    b = ptv.tv1w_2d(cmt, w1t, w2t, max_iters=maxit, method=m)
                    assert a.is_contiguous() and b.stride() == cmt.stride() and a.dtype == torch.float64
                    assert np.array_equal(a.cpu().numpy(), want) and np.array_equal(b.cpu().numpy(), want), case


def test_numpy_surface_and_torch_weight_casts(ptv):
    """numpy tv1w_2d: a Fortran-ordered float64 result equal to the port; torch weights of another dtype and device are moved to x's."""
    import torch
    Y = O.gen_cfg2(70, 45, seed=4, block=8)
    W1, W2 = maps("zeros", 70, 45, seed=5)
    for alg, m in METHODS.items():
        want, _ = port.cp2w_tv(Y, W1, W2, alg, 300)
        got = ptv.tv1w_2d(Y, W1, W2, max_iters=300, method=m)
        assert got.flags.f_contiguous and got.dtype == np.float64 and np.array_equal(got, want), m
        w1c, w2c = torch.tensor(W1, dtype=torch.float32), torch.tensor(W2, dtype=torch.float32)          # CPU float32
        want32w, _ = port.cp2w_tv(Y, w1c.double().numpy(), w2c.double().numpy(), alg, 300)
        t = ptv.tv1w_2d(torch.tensor(Y, device="cuda"), w1c, w2c, max_iters=300, method=m)
        assert np.array_equal(t.cpu().numpy(), want32w), m


def test_constant_maps_equal_tv1_2d(ptv):
    """Maps equal to lambda give the product's own unweighted solver bit for bit, float64 and float32, numpy and torch."""
    import torch
    Y = O.gen_cfg2(128, 96, seed=11, block=16)
    lam = 0.2
    W1, W2 = np.full((127, 96), lam), np.full((128, 95), lam)
    Yb = np.stack([Y, O.gen_cfg2(128, 96, seed=12, block=8)])
    Wb1, Wb2 = np.stack([W1, W1]), np.stack([W2, W2])
    for alg, m in METHODS.items():
        assert np.array_equal(ptv.tv1w_2d(Y, W1, W2, max_iters=400, method=m), ptv.tv1_2d(Y, lam, max_iters=400, method=m)), m
        for dt in (np.float64, np.float32):
            a = ptv.tv1w_2d_batched(Yb.astype(dt), Wb1, Wb2, max_iters=400, method=m)
            b = ptv.tv1_2d_batched(Yb.astype(dt), lam, max_iters=400, method=m)
            assert a.dtype == dt and np.array_equal(a, b), (m, dt)
        tb = torch.tensor(Yb, device="cuda")
        a = ptv.tv1w_2d_batched(tb, torch.tensor(Wb1), torch.tensor(Wb2), max_iters=400, method=m)
        assert torch.equal(a, ptv.tv1_2d_batched(tb, lam, max_iters=400, method=m)), m


def test_batch_mixing_stopped_and_running_images(ptv):
    """A constant image (stops after one iteration) among running images, each with its own maps: every image equals its own single
    solve and keeps its own iteration count, through proxtv_CP2W_TV_batched_f64, numpy and torch tv1w_2d_batched."""
    import torch
    H, W = 40, 36
    imgs = [O.gen_cfg2(H, W, seed=20 + b, block=4) for b in range(4)]
    imgs.insert(1, np.full((H, W), 0.75))
    B = len(imgs)
    ws = [maps("zeros" if b % 2 else "random", H, W, seed=60 + b) for b in range(B)]
    Yb = np.ascontiguousarray(np.stack(imgs))                                      # (B, H, W) C order
    Wb1 = np.ascontiguousarray(np.stack([w[0] for w in ws])); Wb2 = np.ascontiguousarray(np.stack([w[1] for w in ws]))
    lib = ptv.load()
    for alg, m in METHODS.items():
        wants = [port.cp2w_tv(imgs[b], ws[b][0], ws[b][1], alg, 1500) for b in range(B)]
        out = np.zeros_like(Yb); info = np.zeros(3 * B)
        assert lib.proxtv_CP2W_TV_batched_f64(H, W, B, 1, Yb.ctypes.data, Wb1.ctypes.data, Wb2.ctypes.data, out.ctypes.data, alg, 1500,
                                              info.ctypes.data) == 1
        for b, (want, winfo) in enumerate(wants):
            assert np.array_equal(out[b], want), (m, b)
            assert info[3 * b] == winfo[0] and info[3 * b + 2] == 0, (m, b, info[3 * b], winfo[0])
        assert info[3] == 2 and len({info[3 * b] for b in range(B)}) > 1
        got = ptv.tv1w_2d_batched(Yb, Wb1, Wb2, max_iters=1500, method=m)
        assert got.dtype == np.float64 and got.flags.c_contiguous and np.array_equal(got, out)
        gt = ptv.tv1w_2d_batched(torch.tensor(Yb, device="cuda"), torch.tensor(Wb1), torch.tensor(Wb2), max_iters=1500, method=m)
        assert np.array_equal(gt.cpu().numpy(), out)
        cm = torch.tensor(np.ascontiguousarray(Yb.transpose(0, 2, 1)), device="cuda").transpose(1, 2)   # per-image column-major
        gc = ptv.tv1w_2d_batched(cm, torch.tensor(Wb1), torch.tensor(Wb2), max_iters=1500, method=m)
        assert gc.stride() == cm.stride() and np.array_equal(gc.cpu().numpy(), out)


def test_float32_close_to_float64(ptv):
    import torch
    Y = O.gen_cfg2(128, 96, seed=2, block=16)
    W1, W2 = maps("zeros", 128, 96, seed=3)
    for alg in (0, 1):
        want, _ = port.cp2w_tv(Y, W1, W2, alg)
        g32 = ptv.tv1w_2d_batched(Y[None].astype(np.float32), W1[None], W2[None], method=METHODS[alg])
        assert g32.dtype == np.float32
        assert relerr(g32[0], want) <= 1e-4, (alg, relerr(g32[0], want))
        t32 = ptv.tv1w_2d(torch.tensor(Y, dtype=torch.float32, device="cuda"), torch.tensor(W1), torch.tensor(W2), method=METHODS[alg])
        assert t32.dtype == torch.float32 and np.array_equal(t32.cpu().numpy(), g32[0])


def test_requires_grad_raises(ptv):
    import torch
    x = torch.randn(16, 12, dtype=torch.float64, device="cuda")
    w1 = torch.rand(15, 12, dtype=torch.float64, device="cuda"); w2 = torch.rand(16, 11, dtype=torch.float64, device="cuda")
    for m in METHODS.values():
        for which in range(3):
            args = [t.clone().requires_grad_(i == which) for i, t in enumerate((x, w1, w2))]
            with pytest.raises(NotImplementedError, match="backward"):
                ptv.tv1w_2d(*args, method=m)
            with pytest.raises(NotImplementedError, match="backward"):
                ptv.tv1w_2d_batched(*[a[None] for a in args], method=m)
            with torch.no_grad():
                assert ptv.tv1w_2d(*args, method=m, max_iters=5).shape == x.shape
                assert ptv.tv1w_2d_batched(*[a[None] for a in args], method=m, max_iters=5).shape == (1,) + x.shape
            det = [a.detach() for a in args]
            assert torch.equal(ptv.tv1w_2d(*det, method=m, max_iters=5), ptv.tv1w_2d(x, w1, w2, method=m, max_iters=5))


def test_dev_entry_point_on_stream(ptv):
    """proxtv_CP2W_TV_dev_f64 on a side stream with info per image; NULL info and a NULL stream are accepted."""
    import torch
    Y = O.gen_cfg2(33, 47, seed=5, block=4)
    W1, W2 = maps("random", 33, 47, seed=9)
    want, winfo = port.cp2w_tv(Y, W1, W2, 1, 0)
    x = torch.tensor(np.ascontiguousarray(Y.T), device="cuda")                    # column-major storage of Y
    w1 = torch.tensor(np.ascontiguousarray(W1.T), device="cuda"); w2 = torch.tensor(np.ascontiguousarray(W2.T), device="cuda")
    p = [C.c_void_p(t.data_ptr()) for t in (x, w1, w2)]
    out = torch.empty_like(x); info = np.zeros(3)
    s = torch.cuda.Stream()
    lib = ptv.load()
    with torch.cuda.stream(s):
        assert lib.proxtv_CP2W_TV_dev_f64(33, 47, 1, 0, *p, C.c_void_p(out.data_ptr()), 1, 0, info.ctypes.data, C.c_void_p(s.cuda_stream)) == 1
        s.synchronize()
    assert np.array_equal(out.cpu().numpy().T, want) and info[0] == winfo[0] and info[2] == 0
    out2 = torch.empty_like(x)
    assert lib.proxtv_CP2W_TV_dev_f64(33, 47, 1, 0, *p, C.c_void_p(out2.data_ptr()), 1, 0, None, None) == 1
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
