"""GPU tests of CondatChambollePock2_TV (cp2.cu): float64 bit for bit equal to the port (tests/cp2_port.c, itself pinned to the
reference by tests/test_cp2_cpu.py), iteration counts included, through every entry point, layout and batch form; float32 close to it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import relerr
from oracle import oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import cp2_port as port  # noqa: E402
import make_cp2_checks as CP  # noqa: E402

pytestmark = pytest.mark.gpu
METHODS = {0: "condat", 1: "chambolle-pock", 2: "chambolle-pock-acc"}


def abi_solve(ptv, Y, lam, alg, maxit):
    """The reference's entry point: (X, info)."""
    Y = np.asfortranarray(Y, dtype=np.float64); X = np.zeros_like(Y, order="F"); info = np.zeros(3)
    rc = ptv.load().CondatChambollePock2_TV(Y.shape[0], Y.shape[1], Y.ctypes.data, float(lam), X.ctypes.data, alg, int(maxit),
                                            info.ctypes.data)
    assert rc == 1 and info[2] == 0, ptv._lib.last_error()
    return X, info


def test_fixture_cases_bitwise(ptv):
    for key, Y, lam, alg, maxit in CP.cases():
        want, winfo = port.cp2_tv(Y, lam, alg, maxit)
        got, ginfo = abi_solve(ptv, Y, lam, alg, maxit)
        assert np.array_equal(got, want), key
        assert ginfo[0] == winfo[0], (key, ginfo[0], winfo[0])


def test_tv1_2d_numpy_512x384(ptv):
    Y = O.gen_cfg2(512, 384, seed=11, block=16)
    for alg, m in METHODS.items():
        want, winfo = port.cp2_tv(Y, 0.2, alg, 200)
        got = ptv.tv1_2d(Y, 0.2, max_iters=200, method=m)
        assert got.flags.f_contiguous and got.dtype == np.float64
        assert np.array_equal(got, want), m
        _, ginfo = abi_solve(ptv, Y, 0.2, alg, 200)
        assert ginfo[0] == winfo[0] == 201


def test_torch_layouts_bitwise(ptv):
    import torch
    Y = O.gen_cfg2(70, 45, seed=4, block=8)
    for alg, m in METHODS.items():
        want, _ = port.cp2_tv(Y, 0.3, alg, 300)
        rm = torch.tensor(np.ascontiguousarray(Y), device="cuda")                 # C order: row_major = 1
        cm = torch.tensor(np.ascontiguousarray(Y.T), device="cuda").t()           # column-major: row_major = 0
        a = ptv.tv1_2d(rm, 0.3, max_iters=300, method=m)
        b = ptv.tv1_2d(cm, 0.3, max_iters=300, method=m)
        assert a.is_contiguous() and b.stride() == cm.stride() and a.dtype == torch.float64
        assert np.array_equal(a.cpu().numpy(), want) and np.array_equal(b.cpu().numpy(), want), m


def test_batch_mixing_stopped_and_running_images(ptv):
    """A constant image (stops after one iteration) among gen_cfg2 images: every image equals its own single solve and keeps its own
    iteration count, through the host batched entry point, the numpy and the torch batched surface."""
    import torch
    H, W = 40, 36
    imgs = [O.gen_cfg2(H, W, seed=20 + b, block=4) for b in range(4)]
    imgs.insert(1, np.full((H, W), 0.75))
    Yb = np.ascontiguousarray(np.stack(imgs))                                      # (B, H, W) C order
    lib = ptv.load()
    for alg, m in METHODS.items():
        wants = [port.cp2_tv(im, 0.1, alg, 1500) for im in imgs]
        out = np.zeros_like(Yb); info = np.zeros(3 * len(imgs))
        assert lib.proxtv_CP2_TV_batched_f64(H, W, len(imgs), 1, Yb.ctypes.data, 0.1, out.ctypes.data, alg, 1500, info.ctypes.data) == 1
        for b, (want, winfo) in enumerate(wants):
            assert np.array_equal(out[b], want), (m, b)
            assert info[3 * b] == winfo[0] and info[3 * b + 2] == 0, (m, b, info[3 * b], winfo[0])
        assert info[3] == 2 and len({info[3 * b] for b in range(len(imgs))}) > 1
        got = ptv.tv1_2d_batched(Yb, 0.1, max_iters=1500, method=m)
        assert got.dtype == np.float64 and np.array_equal(got, out)
        gt = ptv.tv1_2d_batched(torch.tensor(Yb, device="cuda"), 0.1, max_iters=1500, method=m)
        assert np.array_equal(gt.cpu().numpy(), out)


def test_float32_close_to_float64(ptv):
    import torch
    Y = O.gen_cfg2(128, 96, seed=2, block=16)
    for alg in (0, 1):
        want, _ = port.cp2_tv(Y, 0.2, alg)
        g32 = ptv.tv1_2d_batched(Y[None].astype(np.float32), 0.2, method=METHODS[alg])
        assert g32.dtype == np.float32
        assert relerr(g32[0], want) <= 1e-4, (alg, relerr(g32[0], want))
        t32 = ptv.tv1_2d(torch.tensor(Y, dtype=torch.float32, device="cuda"), 0.2, method=METHODS[alg])
        assert t32.dtype == torch.float32 and np.array_equal(t32.cpu().numpy(), g32[0])


def test_methods_agree_like_the_reference(ptv):
    """prox_tv_test.py:106-115 restated (seeded): condat, chambolle-pock, pd and dr at max_iters = 5000 agree within atol 1e-3."""
    rng = np.random.default_rng(106)
    for _ in range(20):
        x = 100 * rng.normal(size=(int(rng.integers(10, 30)), int(rng.integers(10, 30))))
        w = 20 * rng.random()
        sols = [ptv.tv1_2d(x, w, method=m, max_iters=5000) for m in ("dr", "condat", "chambolle-pock", "pd")]
        for s in sols[1:]:
            assert np.allclose(s, sols[0], atol=1e-3)


def test_requires_grad_raises(ptv):
    import torch
    x = torch.randn(16, 12, dtype=torch.float64, device="cuda", requires_grad=True)
    for m in METHODS.values():
        with pytest.raises(NotImplementedError, match="backward"):
            ptv.tv1_2d(x, 0.1, method=m)
        with pytest.raises(NotImplementedError, match="backward"):
            ptv.tv1_2d_batched(x[None], 0.1, method=m)
    with torch.no_grad():
        assert ptv.tv1_2d(x, 0.1, method="condat", max_iters=5).shape == x.shape


def test_dev_entry_point_on_stream(ptv):
    """proxtv_CP2_TV_dev_f64 on a side stream with info per image; NULL info is accepted."""
    import torch
    Y = O.gen_cfg2(33, 47, seed=5, block=4)
    want, winfo = port.cp2_tv(Y, 0.2, 1, 0)
    x = torch.tensor(np.ascontiguousarray(Y.T), device="cuda")                    # column-major storage of Y
    out = torch.empty_like(x); info = np.zeros(3)
    s = torch.cuda.Stream()
    lib = ptv.load()
    with torch.cuda.stream(s):
        assert lib.proxtv_CP2_TV_dev_f64(33, 47, 1, 0, C.c_void_p(x.data_ptr()), 0.2, C.c_void_p(out.data_ptr()), 1, 0,
                                         info.ctypes.data, C.c_void_p(s.cuda_stream)) == 1
        s.synchronize()
    assert np.array_equal(out.cpu().numpy().T, want) and info[0] == winfo[0]
    out2 = torch.empty_like(x)
    assert lib.proxtv_CP2_TV_dev_f64(33, 47, 1, 0, C.c_void_p(x.data_ptr()), 0.2, C.c_void_p(out2.data_ptr()), 1, 0, None, None) == 1
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
