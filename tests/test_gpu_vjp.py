"""GPU tests (-m gpu) of the backward pass of the batched 1D prox (vjp.cu through proxtv_prox_fibers_vjp_dev_*) and of the torch
autograd layer on top of it, held to a BIT-EXACT bar: np.array_equal with the host restatement of the contract (vjp_emu.restate).

In every case y is the library's own forward output (lane engine for >= 1024 unweighted fibers of >= 64 samples, chunked engine
otherwise), so the segmentation the backward reads -- runs of bit-equal neighbours -- is the forward's; test_segmentation_* checks that
assumption against the oracle's jump sets on data with separated levels.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import jumps
from vjp_emu import from_flat, restate, to_flat

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# (nf, len, inc): lengths 1..4096 and 10^6, 1..65536 fibers, partial warps, contiguous and strided
SHAPES = ((1, 1, 1), (7, 2, 1), (7, 3, 7), (1, 31, 1), (7, 32, 1), (33, 33, 3), (7, 64, 7), (1024, 64, 1), (1024, 64, 32),
          (1024, 1000, 1), (1024, 1000, 8), (1024, 4096, 1), (65536, 32, 1), (65536, 64, 64), (7, 1000, 1), (1, 1_000_000, 1))
# (data kind, lam, weighted), cycled through the shapes
CASES = (("blocks", 0.2, False), ("ties", 1.0, False), ("const", 0.5, False), ("ramp", 5.0, False), ("alt", 0.3, False),
         ("offset", 0.2, False), ("blocks", 0.0, False), ("ties", 1e4, False), ("blocks", 0.5, True), ("ties", 0.0, True))


def make(kind, nf, ln, rng):
    if kind == "blocks":
        return np.repeat(rng.normal(0, 1, (nf, ln // 16 + 1)), 16, axis=1)[:, :ln] + rng.normal(0, 0.3, (nf, ln))
    if kind == "ties":
        return np.round(rng.normal(0, 3, (nf, ln)))
    if kind == "const":
        return np.full((nf, ln), 2.5)
    if kind == "ramp":
        return np.tile(np.linspace(-3, 3, ln), (nf, 1)) + rng.normal(0, 0.01, (nf, 1))
    if kind == "alt":
        return np.where(np.arange(ln) % 2 == 0, 1.0, -1.0)[None, :] * np.ones((nf, 1))
    if kind == "offset":
        return 1e6 + rng.normal(0, 1, (nf, ln))
    raise ValueError(kind)


def weights(nf, ln, rng):
    W = rng.uniform(0.05, 1.0, (nf, max(ln - 1, 0)))
    W[rng.random(W.shape) < 0.1] = 0.0
    return W


@pytest.fixture
def lib(ptv):
    """The raw C ABI with the backward's automatic chunking, restored after the test whatever it set."""
    L = ptv.load()
    L.proxtv_vjp_tuning(0)
    yield L
    L.proxtv_vjp_tuning(0)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def forward(lib, x, nf, ln, inc, lam, w):
    """The library's forward over the flat device array x (fibers (nf, ln, inc))."""
    y = torch.empty_like(x)
    f = lib.proxtv_prox_fibers_dev_f32 if x.dtype == torch.float32 else lib.proxtv_prox_fibers_dev_f64
    assert f(_p(x), _p(y), nf, ln, inc, lam, _p(w), None) == 1
    return y


def backward(lib, y, g, nf, ln, inc, lam, w, want_gw, stream=None):
    gx = torch.full_like(y, float("nan"))
    gw = torch.full((nf * max(ln - 1, 0),), float("nan"), dtype=y.dtype, device=y.device) if want_gw else None
    f = lib.proxtv_prox_fibers_vjp_dev_f32 if y.dtype == torch.float32 else lib.proxtv_prox_fibers_vjp_dev_f64
    assert f(_p(y), _p(g), _p(gx), _p(gw), nf, ln, inc, lam, _p(w), stream) == 1, lib.proxtv_last_error()
    return gx, gw


def run_case(lib, nf, ln, inc, kind, lam, weighted, dtype, rng):
    X = make(kind, nf, ln, rng).astype(dtype)
    W = weights(nf, ln, rng).astype(dtype) if weighted else None
    G = rng.normal(0, 1, (nf, ln)).astype(dtype)
    x = torch.from_numpy(to_flat(X, inc)).cuda()
    w = torch.from_numpy(to_flat(W, inc)).cuda() if weighted else None
    g = torch.from_numpy(to_flat(G, inc)).cuda()
    y = forward(lib, x, nf, ln, inc, lam, w)
    Y = from_flat(y.cpu().numpy(), nf, ln, inc)
    want_gx, want_gw = restate(Y, G, lam, W)
    return x, y, g, w, Y, G, W, want_gx, want_gw


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_vjp_equals_restatement(lib, dtype):
    rng = np.random.default_rng(0)
    for si, (nf, ln, inc) in enumerate(SHAPES):
        kind, lam, weighted = CASES[si % len(CASES)]
        if ln == 1_000_000:
            kind, lam, weighted = "blocks", 0.5, False
        x, y, g, w, Y, G, W, want_gx, want_gw = run_case(lib, nf, ln, inc, kind, lam, weighted, dtype, rng)
        for want in (True, False):
            gx, gw = backward(lib, y, g, nf, ln, inc, lam, w, want)
            gxh = from_flat(gx.cpu().numpy(), nf, ln, inc)
            assert np.array_equal(gxh, want_gx), (nf, ln, inc, kind, lam, weighted, want)
            if want:
                gwh = from_flat(gw.cpu().numpy(), nf, ln - 1, inc)
                assert np.array_equal(gwh, want_gw), (nf, ln, inc, kind, lam, weighted)
                # invariants: gx constant on every segment, gw exactly 0 on fused edges
                wpos = (W > 0) if W is not None else np.full(Y[:, 1:].shape, lam > 0)
                fused = (Y[:, 1:] == Y[:, :-1]) & wpos
                assert np.all(gxh[:, 1:][fused] == gxh[:, :-1][fused]) and np.all(gwh[fused] == 0)
        if lam == 0 and not weighted:
            assert np.array_equal(gxh, G)
        gx2, gw2 = backward(lib, y, g, nf, ln, inc, lam, w, True)
        gx1, gw1 = backward(lib, y, g, nf, ln, inc, lam, w, True)
        assert torch.equal(gx1, gx2) and torch.equal(gw1, gw2)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_forced_chunk_lengths(lib, dtype):
    """The work split through the tuning hook: chunks of 1, 3, 32, 1000 rows, whole fibers, and a constant fiber (one carry chain)."""
    rng = np.random.default_rng(1)
    for (nf, ln, inc, kind, lam, weighted) in ((7, 3000, 1, "blocks", 0.3, False), (64, 2000, 32, "ties", 1.0, True),
                                                (1, 200_000, 1, "const", 0.5, False), (33, 1000, 3, "alt", 0.3, False)):
        x, y, g, w, Y, G, W, want_gx, want_gw = run_case(lib, nf, ln, inc, kind, lam, weighted, dtype, rng)
        for chunk in (1, 3, 32, 1000, 10 ** 7):
            lib.proxtv_vjp_tuning(chunk)
            gx, gw = backward(lib, y, g, nf, ln, inc, lam, w, True)
            assert np.array_equal(from_flat(gx.cpu().numpy(), nf, ln, inc), want_gx), (nf, ln, kind, chunk)
            assert np.array_equal(from_flat(gw.cpu().numpy(), nf, ln - 1, inc), want_gw), (nf, ln, kind, chunk)


def separated(nf, ln, rng):
    """Plateaus of 16 samples at levels 3 apart (shuffled) plus noise 0.05: with lam = 0.3 the prox keeps every plateau."""
    lv = np.stack([rng.permutation(ln // 16 + 1) * 3.0 for _ in range(nf)])
    return np.repeat(lv, 16, axis=1)[:, :ln] + rng.normal(0, 0.05, (nf, ln))


@pytest.mark.parametrize("engine", ["lane", "chunked"])
def test_segmentation_is_the_oracle_jump_set(ptv, lib, port, engine):
    """Runs of bit-equal neighbours in the forward's output are exactly the oracle's segments (jumps(x, 1e-9) convention)."""
    rng = np.random.default_rng(2)
    nf, ln, lam = 1024, 256, 0.3
    X = separated(nf, ln, rng)
    prev = ptv.set_engine(engine)
    try:
        Y =ptv.tv1_1d_batched(torch.from_numpy(X).cuda(), lam).cpu().numpy()
        Yw = ptv.tv1w_1d_batched(torch.from_numpy(X).cuda(), torch.full((nf, ln - 1), lam, dtype=torch.float64, device="cuda")).cpu().numpy()
    finally:
        ptv.set_engine(prev)
    for f in range(0, nf, 7):
        want = jumps(port.tv1_linearized(X[f], lam), 1e-9)
        assert np.array_equal(np.flatnonzero(Y[f, 1:] != Y[f, :-1]), want), f
        assert np.array_equal(np.flatnonzero(Yw[f, 1:] != Yw[f, :-1]), jumps(port.tv1_weighted(X[f], np.full(ln - 1, lam)), 1e-9)), f


def test_refusals_write_nothing(lib):
    y = torch.zeros(64, dtype=torch.float64, device="cuda"); g = torch.ones_like(y)
    gx = torch.full_like(y, -7.0); gw = torch.full((63,), -7.0, dtype=torch.float64, device="cuda")
    f = lib.proxtv_prox_fibers_vjp_dev_f64
    for args in ((_p(y), _p(g), _p(gx), _p(gw), -1, 64, 1, 0.5, None), (_p(y), _p(g), _p(gx), _p(gw), 1, -64, 1, 0.5, None),
                 (_p(y), _p(g), _p(gx), _p(gw), 1, 64, 0, 0.5, None), (None, _p(g), _p(gx), _p(gw), 1, 64, 1, 0.5, None),
                 (_p(y), None, _p(gx), _p(gw), 1, 64, 1, 0.5, None), (_p(y), _p(g), None, _p(gw), 1, 64, 1, 0.5, None),
                 (_p(y), _p(g), _p(gx), _p(gw), 1, 64, 1, -0.5, None)):
        assert f(*args, None) == 0
        assert "proxtv_prox_fibers_vjp_dev_f64" in lib.proxtv_last_error().decode()
    torch.cuda.synchronize()
    assert torch.all(gx == -7.0) and torch.all(gw == -7.0)
    assert f(_p(y), _p(g), _p(gx), _p(gw), 0, 64, 1, 0.5, None, None) == 1
    assert f(_p(y), _p(g), _p(gx), _p(gw), 1, 0, 1, 0.5, None, None) == 1
    y32 = y.float(); g32 = g.float(); gx32 = torch.full_like(y32, -7.0)
    assert lib.proxtv_prox_fibers_vjp_dev_f32(_p(y32), _p(g32), _p(gx32), None, 1, 64, 1, -0.5, None, None) == 0
    assert "proxtv_prox_fibers_vjp_dev_f32" in lib.proxtv_last_error().decode()
    torch.cuda.synchronize()
    assert torch.all(gx32 == -7.0)


# ---- torch autograd ----
def test_gradcheck(ptv):
    rng = np.random.default_rng(3)
    X = torch.from_numpy(separated(3, 40, rng)).cuda().requires_grad_()
    lam = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: ptv.tv1_1d_batched(a, b), (X, lam), eps=1e-6, atol=1e-6)
    W = torch.from_numpy(rng.uniform(0.2, 0.4, (3, 39))).cuda().requires_grad_()
    assert torch.autograd.gradcheck(lambda a, b: ptv.tv1w_1d_batched(a, b), (X, W), eps=1e-6, atol=1e-6)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_autograd_equals_c_abi(ptv, lib, dtype):
    rng = np.random.default_rng(4)
    B, L = 1500, 300
    X = torch.from_numpy(make("blocks", B, L, rng)).to(device="cuda", dtype=dtype)
    Wt = torch.from_numpy(weights(B, L, rng)).to(device="cuda", dtype=dtype)
    G = torch.from_numpy(rng.normal(0, 1, (B, L))).to(device="cuda", dtype=dtype)
    # scalar penalty as a 0-dim tensor
    x = X.clone().requires_grad_(); lam = torch.tensor(0.4, dtype=torch.float64, device="cuda", requires_grad=True)
    y = ptv.tv1_1d_batched(x, lam)
    with torch.no_grad():
        y0 = ptv.tv1_1d_batched(X, 0.4)
    assert y.grad_fn is not None and y0.grad_fn is None and torch.equal(y.detach(), y0)
    y.backward(G)
    gx, gw = backward(lib, y0.reshape(-1), G.reshape(-1), B, L, 1, 0.4, None, True)
    assert torch.equal(x.grad, gx.reshape(B, L))
    assert lam.grad.dtype == torch.float64 and lam.grad.shape == ()
    assert torch.equal(lam.grad, gw.sum(dtype=torch.float64))
    # per-edge weights
    x = X.clone().requires_grad_(); w = Wt.clone().requires_grad_()
    y = ptv.tv1w_1d_batched(x, w)
    with torch.no_grad():
        y0 = ptv.tv1w_1d_batched(X, Wt)
    assert torch.equal(y.detach(), y0)
    y.backward(G)
    gx, gw = backward(lib, y0.reshape(-1), G.reshape(-1), B, L, 1, 0.0, Wt.reshape(-1), True)
    assert torch.equal(x.grad, gx.reshape(B, L)) and torch.equal(w.grad, gw.reshape(B, L - 1))


def test_autograd_views_streams_and_float_penalty(ptv, lib):
    rng = np.random.default_rng(5)
    B, L = 64, 500
    base = torch.from_numpy(make("blocks", L, 2 * B, rng)).to(device="cuda", dtype=torch.float32)
    G = torch.from_numpy(rng.normal(0, 1, (B, L))).to(device="cuda", dtype=torch.float32)
    xv = base.t()[::2]                                    # a (B, L) view that is not contiguous
    assert not xv.is_contiguous()
    leaf = base.clone().requires_grad_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        y = ptv.tv1_1d_batched(leaf.t()[::2], 0.5)        # python float: gradient for x only
        y.backward(G)
    s.synchronize()
    y0 = ptv.tv1_1d_batched(xv.contiguous(), 0.5)
    assert torch.equal(y.detach(), y0)
    gx, _ = backward(lib, y0.reshape(-1), G.reshape(-1), B, L, 1, 0.5, None, False)
    want = torch.zeros_like(base).t().contiguous()
    want[::2] = gx.reshape(B, L)
    assert torch.equal(leaf.grad, want.t())


def test_no_grad_path_saves_nothing(ptv):
    x = torch.randn(8, 100, dtype=torch.float64, device="cuda")
    y = ptv.tv1_1d_batched(x, 0.3)                        # x does not require grad
    assert y.grad_fn is None
    xr = x.clone().requires_grad_()
    with torch.no_grad():
        y2 = ptv.tv1_1d_batched(xr, 0.3)
    assert y2.grad_fn is None and torch.equal(y, y2)
    w = torch.full((8, 99), 0.3, dtype=torch.float64, device="cuda")
    assert ptv.tv1w_1d_batched(x, w).grad_fn is None
