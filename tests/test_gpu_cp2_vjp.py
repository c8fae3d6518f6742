"""GPU tests of the converged 2D TV-L1 backward (tv1_2d / tv1w_2d and their batched forms with backward='converged',
proxtv_CP2_TV_* / proxtv_CP2W_TV_* record and vjp, DESIGN.md section 15.2): the recorded forward is the unrecorded one bit for bit, the
tape is the host fusion rule on the port's duals, the backward agrees with the float64 host restatement (tests/cp2_vjp_host.py) in both
storage orders and from run to run, finite differences through the GPU forward, projection properties, the 1D backward where the
problem separates, the labelling under clusters that cross every tile, and the refusals."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cp2_vjp_host as H  # noqa: E402

pytestmark = pytest.mark.gpu
METHODS = {0: "condat", 1: "chambolle-pock"}


def _t(a, dtype=None, order="C"):
    import torch
    dt = dtype or torch.float64
    t = torch.as_tensor(np.ascontiguousarray(a)).to(device="cuda", dtype=dt)
    return t if order == "C" else t.transpose(-2, -1).contiguous().transpose(-2, -1)


def piecewise(M, N, seed):
    return O.gen_cfg2(M, N, seed=seed, block=8) + 0.05 * np.random.default_rng(seed).normal(size=(M, N))


def _solve(ptv, xin, W1, W2, lam, alg, maxit, record):
    """(X, info, tape) of the raw dev / record_dev call on xin (batch, M, N) in its own layout."""
    import torch
    batch, M, N = xin.shape
    row_major = 1 if xin.stride(-1) == 1 else 0
    geom = (M, N, batch, row_major, alg, maxit)
    tape = torch.empty(int(ptv.load().proxtv_CP2_TV_tape_bytes(M, N, batch)), dtype=torch.uint8, device="cuda") if record else None
    out = torch.empty_strided(xin.shape, xin.stride(), dtype=xin.dtype, device="cuda")
    info = np.zeros(3 * batch)
    entry, pen = ("CP2W_TV", (W1, W2)) if W1 is not None else ("CP2_TV", (lam,))
    args = (M, N, batch, row_major, xin, *pen, out, alg, maxit, info)
    if record:
        ptv._dev_call(entry + "_record_dev", xin, *args, tape, tape.numel(), info=info)
    else:
        ptv._dev_call(entry + "_dev", xin, *args, info=info)
    torch.cuda.synchronize()
    return out, info, tape


def _bits(tape, n):
    """The two bitsets of a tape (F, S), n bits each, in storage order."""
    raw = tape.cpu().numpy()
    sb = ((n + 31) // 32 * 4 + 255) // 256 * 256
    f = np.unpackbits(raw[256:256 + sb], bitorder="little")[:n].astype(bool)
    s = np.unpackbits(raw[256 + sb:256 + 2 * sb], bitorder="little")[:n].astype(bool)
    return f, s


def _index_bits(tape, M, N, batch, row_major):
    """The tape as index-order fused maps f1 (batch, M-1, N) (axis 0) and f2 (batch, M, N-1) (axis 1)."""
    f, s = _bits(tape, M * N * batch)
    if row_major:       # storage (b, i, j): F = axis 1, S = axis 0
        F = f.reshape(batch, M, N); S = s.reshape(batch, M, N)
        return S[:, :-1, :], F[:, :, :-1]
    F = f.reshape(batch, N, M).transpose(0, 2, 1); S = s.reshape(batch, N, M).transpose(0, 2, 1)
    return F[:, :-1, :], S[:, :, :-1]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("order", ["C", "F"])
def test_recorded_forward_is_unrecorded(ptv, weighted, dtype, order):
    """X and info bit for bit, on a batch that mixes a constant image with running ones."""
    import torch
    dt = torch.float64 if dtype == "f64" else torch.float32
    M, N = 70, 45
    Y = np.stack([piecewise(M, N, 1), np.full((M, N), 0.7), np.random.default_rng(2).normal(size=(M, N))])
    rng = np.random.default_rng(3)
    xin = _t(Y, dt, order)
    W1 = _t(rng.uniform(0, 0.5, (3, M - 1, N)), dt, order) if weighted else None
    W2 = _t(rng.uniform(0, 0.5, (3, M, N - 1)), dt, order) if weighted else None
    for alg in (0, 1):
        a, ia, _ = _solve(ptv, xin, W1, W2, 0.3, alg, 0, False)
        b, ib, _ = _solve(ptv, xin, W1, W2, 0.3, alg, 0, True)
        assert torch.equal(a, b) and np.array_equal(ia, ib)
        assert ia[3] == 2                                   # the constant image stops at once


@pytest.mark.parametrize("weighted", [False, True])
def test_tape_is_the_host_rule(ptv, weighted):
    """float64: the tape's bits are the fusion rule applied to the port's final duals and X, in both storage orders."""
    M, N, lam = 40, 36, 0.4
    Y = piecewise(M, N, 4)
    rng = np.random.default_rng(5)
    W1, W2 = (rng.uniform(0, 0.6, (M - 1, N)), rng.uniform(0, 0.6, (M, N - 1))) if weighted else H.weights(M, N, lam)
    for alg in (0, 1):
        X, U1, U2, info = H.solve(Y, W1, W2, alg)
        f1, f2 = H.fused(X, U1, U2, W1, W2)
        for order in ("C", "F"):
            wt = (_t(W1[None], order=order), _t(W2[None], order=order)) if weighted else (None, None)
            out, ginfo, tape = _solve(ptv, _t(Y[None], order=order), *wt, lam, alg, 0, True)
            assert np.array_equal(out[0].cpu().numpy(), X) and ginfo[0] == info[0]
            g1, g2 = _index_bits(tape, M, N, 1, order == "C")
            assert np.array_equal(g1[0], f1) and np.array_equal(g2[0], f2), (alg, order)


def _grads(ptv, Y, lam, W, alg, dtype, order, G, maxit=0):
    """(y, gx, gw) through autograd: gw = (glam or gW1, gW2) as numpy float64."""
    import torch
    x = _t(Y, dtype, order).requires_grad_(True)
    batched = Y.ndim == 3
    if W is None:
        w = torch.tensor(lam, dtype=torch.float64, device="cuda", requires_grad=True)
        f = ptv.tv1_2d_batched if batched else ptv.tv1_2d
        y = f(x, w, max_iters=maxit, method=METHODS[alg], backward="converged")
        ws = (w,)
    else:
        w1 = _t(W[0], dtype, order).requires_grad_(True); w2 = _t(W[1], dtype, order).requires_grad_(True)
        f = ptv.tv1w_2d_batched if batched else ptv.tv1w_2d
        y = f(x, w1, w2, max_iters=maxit, method=METHODS[alg], backward="converged")
        ws = (w1, w2)
    y.backward(_t(G, dtype, order))
    return y.detach(), x.grad, [v.grad for v in ws]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_backward_against_host(ptv, weighted, dtype):
    """gx within 1e-12 (sum over C of |g|) / |C| (plus the storage rounding) of the host restatement on the tape's partition; gw the
    contract's formula of that gx exactly; glam within 1e-12; the same bits in both orders and from run to run."""
    import torch
    dt = torch.float64 if dtype == "f64" else torch.float32
    eps = np.finfo(np.float64 if dtype == "f64" else np.float32).eps
    B, M, N, lam = 3, 50, 43, 0.35
    Y = np.stack([piecewise(M, N, 10 + b) for b in range(B)])
    rng = np.random.default_rng(7)
    W = (rng.uniform(0, 0.5, (B, M - 1, N)), rng.uniform(0, 0.5, (B, M, N - 1))) if weighted else None
    G = rng.normal(size=Y.shape)
    for alg in (0, 1):
        runs = [_grads(ptv, Y, lam, W, alg, dt, order, G) for order in ("C", "F", "C")]
        y, gx, gw = runs[0]
        for _, gx2, gw2 in runs[1:]:
            assert torch.equal(gx, gx2) and all(torch.equal(a, b) for a, b in zip(gw, gw2))
        # the tape of this forward, for the host's partition
        xin = _t(Y, dt, "C")
        Wt = (_t(W[0], dt), _t(W[1], dt)) if weighted else (None, None)
        _, _, tape = _solve(ptv, xin, *Wt, lam, alg, 0, True)
        f1s, f2s = _index_bits(tape, M, N, B, 1)
        Gq = _t(G, dt).double().cpu().numpy()
        Xn, gxn = y.double().cpu().numpy(), gx.double().cpu().numpy()
        glam, tot = np.zeros(2), 0.0
        for b in range(B):
            hx, _, _, _ = H.vjp(Xn[b], f1s[b], f2s[b], Gq[b])
            scale = H.cluster_abs_mean(f1s[b], f2s[b], Gq[b])
            assert np.all(np.abs(gxn[b] - hx) <= 1e-12 * scale + eps * np.abs(hx)), (alg, b)
            # the edge gradients from the device's gx, by the contract's formula
            gw1 = np.where(f1s[b], 0.0, np.sign(Xn[b, 1:] - Xn[b, :-1]) * (gxn[b, :-1] - gxn[b, 1:])).astype(Gq.dtype if dtype == "f64" else np.float32)
            gw2 = np.where(f2s[b], 0.0, np.sign(Xn[b, :, 1:] - Xn[b, :, :-1]) * (gxn[b, :, :-1] - gxn[b, :, 1:])).astype(gw1.dtype)
            if weighted:
                assert np.array_equal(gw[0][b].cpu().numpy(), gw1) and np.array_equal(gw[1][b].cpu().numpy(), gw2)
            else:
                glam += [gw1.astype(np.float64).sum(), gw2.astype(np.float64).sum()]
                tot += np.abs(gw1).astype(np.float64).sum() + np.abs(gw2).astype(np.float64).sum()
        if not weighted:
            assert abs(float(gw[0]) - glam.sum()) <= 1e-12 * max(tot, 1.0)


def _fd(f, x, d, eps=1e-6):
    return (f(x + eps * d) - f(x - eps * d)) / (2 * eps)


@pytest.mark.parametrize("alg", [0, 1])
def test_finite_differences_through_the_gpu_forward(ptv, alg):
    """48 x 40 float64: <g, J d> by central differences against <gx, d>, d(lambda), and per-edge weight maps."""
    import torch
    M, N = 48, 40
    Y = piecewise(M, N, 20)
    rng = np.random.default_rng(21)
    G = rng.normal(size=(M, N)); D = rng.normal(size=(M, N))
    m = METHODS[alg]
    _, gx, (gw,) = _grads(ptv, Y, 0.3, None, alg, torch.float64, "C", G)
    Gt = _t(G)
    with torch.no_grad():
        fx = lambda x: float((Gt * ptv.tv1_2d(x, 0.3, method=m)).sum())  # noqa: E731
        assert abs(_fd(fx, _t(Y), _t(D)) - float((gx * _t(D)).sum())) < 1e-6
        fl = lambda lam: float((Gt * ptv.tv1_2d(_t(Y), lam, method=m)).sum())  # noqa: E731
        assert abs(_fd(fl, 0.3, 1.0) - float(gw)) < 1e-6
    W = (rng.uniform(0.1, 0.5, (M - 1, N)), rng.uniform(0.1, 0.5, (M, N - 1)))
    _, gx, (g1, g2) = _grads(ptv, Y, None, W, alg, torch.float64, "C", G)
    D1, D2 = rng.normal(size=W[0].shape), rng.normal(size=W[1].shape)
    with torch.no_grad():
        fw = lambda s: float((Gt * ptv.tv1w_2d(_t(Y), _t(W[0] + s * D1), _t(W[1] + s * D2), method=m)).sum())  # noqa: E731
        want = float((g1 * _t(D1)).sum() + (g2 * _t(D2)).sum())
        assert abs(_fd(fw, 0.0, 1.0) - want) < 1e-6


def test_gradcheck_small(ptv):
    import torch
    x = _t(piecewise(9, 7, 30)).requires_grad_(True)
    w = torch.tensor(0.25, dtype=torch.float64, device="cuda", requires_grad=True)
    f = lambda x, w: ptv.tv1_2d(x, w, method="condat", backward="converged")  # noqa: E731
    assert torch.autograd.gradcheck(f, (x, w), eps=1e-6, atol=1e-5, rtol=1e-4)


def _vjp_raw(ptv, out, tape, g):
    import torch
    batch, M, N = out.shape
    gY = torch.empty_like(g)
    ptv._dev_call("CP2_TV_vjp_dev", g, M, N, batch, 1, tape, out, g, gY, None)
    return gY


def test_projection_properties(ptv):
    """J gx = gx, <J u, v> = <u, J v>, and sum gx = sum g per image."""
    import torch
    B, M, N = 2, 64, 50
    Y = np.stack([piecewise(M, N, 40 + b) for b in range(B)])
    out, _, tape = _solve(ptv, _t(Y), None, None, 0.3, 0, 0, True)
    rng = np.random.default_rng(41)
    u, v = _t(rng.normal(size=Y.shape)), _t(rng.normal(size=Y.shape))
    Ju, Jv = _vjp_raw(ptv, out, tape, u), _vjp_raw(ptv, out, tape, v)
    assert torch.allclose(_vjp_raw(ptv, out, tape, Ju), Ju, rtol=0, atol=1e-14)
    assert abs(float((Ju * v).sum() - (u * Jv).sum())) < 1e-11
    assert torch.allclose(Ju.sum(dim=(1, 2)), u.sum(dim=(1, 2)), rtol=0, atol=1e-11)


def test_separable_problems_are_the_1d_backward(ptv):
    """w_row = 0 separates the columns: per column the gradients of tv1w_1d_batched's backward within 1e-12; M == 1 and N == 1 are
    tv1_1d_batched's."""
    import torch
    M, N = 40, 6
    Y = piecewise(M, N, 50)
    rng = np.random.default_rng(51)
    G = rng.normal(size=(M, N))
    W1 = rng.uniform(0.1, 0.4, (M - 1, N))
    y, gx, (g1, g2) = _grads(ptv, Y, None, (W1, np.zeros((M, N - 1))), 0, torch.float64, "C", G)
    xc = _t(Y.T.copy()).requires_grad_(True); wc = _t(W1.T.copy()).requires_grad_(True)
    yc = ptv.tv1w_1d_batched(xc, wc)
    yc.backward(_t(G.T.copy()))
    assert torch.allclose(y.t(), yc.detach(), rtol=0, atol=1e-6)
    assert torch.allclose(gx.t(), xc.grad, rtol=0, atol=1e-12) and torch.allclose(g1.t(), wc.grad, rtol=0, atol=1e-12)
    for shape in ((1, 57), (57, 1)):
        Y1 = np.random.default_rng(52).normal(size=shape)
        G1 = np.random.default_rng(53).normal(size=shape)
        _, gx, (gw,) = _grads(ptv, Y1, 0.3, None, 0, torch.float64, "C", G1)
        xr = _t(Y1.reshape(1, -1)).requires_grad_(True)
        wr = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
        ptv.tv1_1d_batched(xr, wr).backward(_t(G1.reshape(1, -1)))
        assert torch.allclose(gx.reshape(1, -1), xr.grad, rtol=0, atol=1e-12)
        assert abs(float(gw) - float(wr.grad)) < 1e-12


def test_serpentine_cluster_crosses_every_tile(ptv):
    """Zero walls carve one serpentine corridor through a 1024^2 image; huge weights keep every dual below its bound, so the whole
    corridor is one cluster: gx is the image mean of g everywhere, in both orders."""
    import torch
    M = N = 1024
    W1 = np.zeros((M - 1, N)); W2 = np.full((M, N - 1), 1e9)
    W1[0::2, -1] = 1e9; W1[1::2, 0] = 1e9                 # row i joins row i + 1 at its right end (i even) or left end (i odd)
    G = np.random.default_rng(60).normal(size=(M, N))
    Y = np.random.default_rng(61).normal(size=(M, N))
    for order in ("C", "F"):
        _, gx, (g1, g2) = _grads(ptv, Y, None, (W1, W2), 0, torch.float64, order, G, maxit=20)
        assert torch.allclose(gx, torch.full_like(gx, G.mean()), rtol=1e-12, atol=1e-15)
        assert float(g1.abs().max()) == 0 and float(g2.abs().max()) == 0
    _, gx, (gw,) = _grads(ptv, Y, 1e9, None, 1, torch.float64, "F", G, maxit=20)
    assert torch.allclose(gx, torch.full_like(gx, G.mean()), rtol=1e-12, atol=1e-15) and float(gw) == 0


@pytest.mark.parametrize("shape,dtype", [((1, 4096, 4096), "f64"), ((8, 2048, 2048), "f32")])
def test_full_size(ptv, shape, dtype):
    """Full-size backward: deterministic, and its projection properties (sum gx = sum g per image, J gx = gx)."""
    import torch
    dt = torch.float64 if dtype == "f64" else torch.float32
    g = torch.Generator(device="cuda").manual_seed(70)
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float64).to(dt)
    G = torch.randn(shape, generator=g, device="cuda", dtype=torch.float64).to(dt)
    out, _, tape = _solve(ptv, x, None, None, 0.3, 0, 200, True)
    a, b = _vjp_raw(ptv, out, tape, G), _vjp_raw(ptv, out, tape, G)
    assert torch.equal(a, b)
    tol = 1e-9 if dtype == "f64" else 1e-2
    assert torch.allclose(a.double().sum(dim=(1, 2)), G.double().sum(dim=(1, 2)), rtol=0, atol=tol)
    assert torch.allclose(_vjp_raw(ptv, out, tape, a), a, rtol=0, atol=1e-14 if dtype == "f64" else 1e-6)


def test_errors(ptv):
    """backward='converged' refuses the accelerated method; the default still raises under grad; a tape of another kind is refused."""
    import torch
    x = torch.randn(16, 12, dtype=torch.float64, device="cuda", requires_grad=True)
    with pytest.raises(NotImplementedError, match="converged"):
        ptv.tv1_2d(x, 0.1, method="chambolle-pock-acc", backward="converged")
    with pytest.raises(NotImplementedError, match="backward"):
        ptv.tv1_2d(x, 0.1, method="condat")
    out, _, tape = _solve(ptv, x.detach()[None], None, None, 0.1, 0, 30, True)
    g = torch.ones_like(out)
    lib = ptv.load()
    gY = torch.full_like(out, -7.0)
    assert lib.proxtv_CP2_TV_vjp_dev_f64(16, 12, 1, 0, tape.data_ptr(), out.data_ptr(), g.data_ptr(), gY.data_ptr(), None, None) == 0
    assert "storage order" in ptv._lib.last_error()
    assert lib.proxtv_CP2_TV_vjp_dev_f64(12, 16, 1, 1, tape.data_ptr(), out.data_ptr(), g.data_ptr(), gY.data_ptr(), None, None) == 0
    assert "shape" in ptv._lib.last_error()
    assert lib.proxtv_CP2W_TV_vjp_dev_f64(16, 12, 1, 1, tape.data_ptr(), out.data_ptr(), g.data_ptr(), gY.data_ptr(), None, None, None,
                                          None) == 0
    assert "unweighted" in ptv._lib.last_error()
    gf = torch.ones_like(out, dtype=torch.float32)
    assert lib.proxtv_CP2_TV_vjp_dev_f32(16, 12, 1, 1, tape.data_ptr(), gf.data_ptr(), gf.data_ptr(), gf.data_ptr(), None, None) == 0
    assert "dtype" in ptv._lib.last_error()
    bad = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    assert lib.proxtv_CP2_TV_vjp_dev_f64(16, 12, 1, 1, bad.data_ptr(), out.data_ptr(), g.data_ptr(), gY.data_ptr(), None, None) == 0
    assert "not a CP2_TV tape" in ptv._lib.last_error()
    assert float(gY.min()) == -7.0 and float(gY.max()) == -7.0
