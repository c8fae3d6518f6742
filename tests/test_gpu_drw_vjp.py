"""GPU tests (-m gpu) of the DR2L1W_TV backward pass (DESIGN.md section 12): the recorded forward, the unrolled backward and the torch
autograd path of tv1w_2d.

Bars:
  * recorded forward == proxtv_DR2L1W_TV_dev_* bit for bit on every engine (seq, auto, chunked), float64 and float32, 1 / 2 / 35
    iterations, N < 64 and N >= 64 (the two row routes), odd sizes, M == 1, N == 1 and 4096^2; every recorded pass's tape == the
    host forward's (drw_vjp_emu.forward) on dyadic float64 inputs, and so is the output;
  * backward == the host restatement driven by the device's own tape (drw_vjp_emu.backward_from_tapes): gW1 and gW2 bit for bit, gY
    to 1e-12 relative (float64) / 1e-5 (float32) -- only the start value term's sum order differs; two identical calls are bit-equal
    and NULL weight maps leave gY unchanged;
  * refusals write nothing; autograd: gradcheck, directional differences, forward bit-equal to the no-grad call, each input alone,
    mixed dtypes, expanded weights, views, streams.
"""
import ctypes as C

import numpy as np
import pytest

import drw_vjp_emu as E
from conftest import relerr
from test_gpu_dr2_vjp import kink_free_difference
from test_gpu_lane import dyadic

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture
def lib(ptv):
    return ptv.load()


@pytest.fixture
def engine(ptv):
    prev = ptv.set_engine("auto")
    ptv.set_engine(prev)
    yield ptv.set_engine
    ptv.set_engine(prev)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _st(stream=None):
    return C.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def problem(shape, seed, dt, zeros=0.15):
    """Dyadic image and weights (multiples of 1/256, some zero), numpy (M, N), (M-1, N), (M, N-1)."""
    M, N = shape
    Y = dyadic((1, M, N), seed, np.float64)[0]
    rng = np.random.default_rng(seed + 100)
    W1 = np.round(rng.uniform(0.05, 0.6, (M - 1, N)) * 256) / 256
    W2 = np.round(rng.uniform(0.05, 0.6, (M, N - 1)) * 256) / 256
    W1[rng.random(W1.shape) < zeros] = 0.0
    W2[rng.random(W2.shape) < zeros] = 0.0
    return Y.astype(dt), W1.astype(dt), W2.astype(dt)


def colmajor(A, dt=None):
    """numpy (R, C) -> the device buffer of its column-major storage: a contiguous (C, R) tensor."""
    T = torch.float32 if (dt or A.dtype) == np.float32 else torch.float64
    return torch.tensor(np.ascontiguousarray(np.asarray(A).T), dtype=T, device="cuda")


def natural(t):
    return t.cpu().numpy().T


def record(lib, Yt, W1t, W2t, M, N, maxit, stream=None):
    out = torch.full_like(Yt, float("nan"))
    nb = lib.proxtv_DR2L1W_TV_tape_bytes(M, N, maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    f = lib.proxtv_DR2L1W_TV_record_dev_f32 if Yt.dtype == torch.float32 else lib.proxtv_DR2L1W_TV_record_dev_f64
    assert f(M, N, _p(Yt), _p(W1t), _p(W2t), _p(out), maxit, _p(tape), nb, C.c_void_p(info.ctypes.data), _st(stream)) == 1, \
        lib.proxtv_last_error()
    assert info[2] == 0
    return out, tape


def solve(lib, Yt, W1t, W2t, M, N, maxit):
    out = torch.full_like(Yt, float("nan"))
    info = np.zeros(3)
    f = lib.proxtv_DR2L1W_TV_dev_f32 if Yt.dtype == torch.float32 else lib.proxtv_DR2L1W_TV_dev_f64
    f(M, N, _p(Yt), _p(W1t), _p(W2t), _p(out), maxit, C.c_void_p(info.ctypes.data), _st())
    assert info[2] != 3, lib.proxtv_last_error()
    return out


def vjp(lib, tape, gout, M, N, maxit, want1=True, want2=True, stream=None):
    gY = torch.full_like(gout, float("nan"))
    gW1 = torch.full((N, M - 1), float("nan"), dtype=gout.dtype, device="cuda") if want1 else None
    gW2 = torch.full((N - 1, M), float("nan"), dtype=gout.dtype, device="cuda") if want2 else None
    f = lib.proxtv_DR2L1W_TV_vjp_dev_f32 if gout.dtype == torch.float32 else lib.proxtv_DR2L1W_TV_vjp_dev_f64
    assert f(M, N, maxit, _p(tape), _p(gout), _p(gY), _p(gW1), _p(gW2), _st(stream)) == 1, lib.proxtv_last_error()
    return gY, gW1, gW2


def check_backward(lib, tape, G, M, N, maxit, what):
    """Device backward against the restatement driven by the device's own tape."""
    dt = G.dtype
    gY, gW1, gW2 = vjp(lib, tape, colmajor(G), M, N, maxit)
    hY, h1, h2 = E.backward_from_tapes(E.device_pass_tapes(tape.cpu().numpy(), M, N, maxit), G, maxit)
    assert np.array_equal(natural(gW1), h1), what
    assert np.array_equal(natural(gW2), h2), what
    assert relerr(natural(gY), hY) <= (1e-12 if dt == np.float64 else 1e-5), what
    return gY, gW1, gW2


SHAPES = [(37, 50), (45, 129), (64, 64), (1, 70), (70, 1), (1, 1)]


@pytest.mark.parametrize("maxit", [1, 2, 35])
def test_recorded_forward_tapes_and_backward(lib, engine, port, maxit):
    """Every engine and dtype: out == proxtv_DR2L1W_TV_dev_* bit for bit, the backward == the tape-driven restatement; float64 also:
    out and every pass's tape == the host forward's."""
    it_arg = 0 if maxit == 35 else maxit
    for si, (M, N) in enumerate(SHAPES):
        Y64, W1_64, W2_64 = problem((M, N), 3 + si, np.float64)
        want, passes = E.forward(port, Y64, W1_64, W2_64, maxit)
        host_tapes = E.pass_tapes(passes, W1_64, W2_64)
        for dt in (np.float64, np.float32):
            Y, W1, W2 = Y64.astype(dt), W1_64.astype(dt), W2_64.astype(dt)
            Yt, W1t, W2t = colmajor(Y), colmajor(W1), colmajor(W2)
            G = np.random.default_rng(si).normal(size=(M, N)).astype(dt)
            for eng in ("seq", "auto", "chunked"):
                engine(eng)
                what = ((M, N), maxit, np.dtype(dt).name, eng)
                out, tape = record(lib, Yt, W1t, W2t, M, N, it_arg)
                assert torch.equal(out, solve(lib, Yt, W1t, W2t, M, N, it_arg)), what
                if dt == np.float64:
                    assert np.array_equal(natural(out), want), what
                    dev_tapes = E.device_pass_tapes(tape.cpu().numpy(), M, N, maxit)
                    for p, ((F, U), (Fh, Uh)) in enumerate(zip(dev_tapes, host_tapes)):
                        assert np.array_equal(F, Fh) and np.array_equal(U, Uh), what + (p,)
                check_backward(lib, tape, G, M, N, it_arg, what)


def test_recorded_forward_4096(lib, engine):
    M = N = 4096
    Y, W1, W2 = problem((M, N), 5, np.float64)
    for dt in (np.float64, np.float32):
        Yt, W1t, W2t = colmajor(Y, dt), colmajor(W1, dt), colmajor(W2, dt)
        for eng in ("auto", "seq") if dt == np.float64 else ("auto",):
            engine(eng)
            out, tape = record(lib, Yt, W1t, W2t, M, N, 0)
            assert torch.equal(out, solve(lib, Yt, W1t, W2t, M, N, 0)), (np.dtype(dt).name, eng)
            del tape
    assert lib.proxtv_DR2L1W_TV_tape_bytes(M, N, 35) == 256 + 72 * 2 * (M * N // 32 * 4)


def test_backward_deterministic_and_null_maps(lib, port):
    M, N = 72, 96
    Y, W1, W2 = problem((M, N), 9, np.float64)
    Yt, W1t, W2t = colmajor(Y), colmajor(W1), colmajor(W2)
    _, tape = record(lib, Yt, W1t, W2t, M, N, 5)
    g = torch.randn_like(Yt)
    a = vjp(lib, tape, g, M, N, 5)
    b = vjp(lib, tape, g, M, N, 5)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for w1, w2 in ((False, False), (True, False), (False, True)):
        c = vjp(lib, tape, g, M, N, 5, w1, w2)
        assert torch.equal(c[0], a[0]), (w1, w2)
        assert (not w1 or torch.equal(c[1], a[1])) and (not w2 or torch.equal(c[2], a[2]))


def test_refusals_write_nothing(lib):
    M, N, K = 40, 70, 3
    Y, W1, W2 = problem((M, N), 2, np.float64)
    Yt, W1t, W2t = colmajor(Y), colmajor(W1), colmajor(W2)
    _, tape = record(lib, Yt, W1t, W2t, M, N, K)
    nb = lib.proxtv_DR2L1W_TV_tape_bytes(M, N, K)
    assert nb == 256 + (2 * K + 2) * 2 * (((M * N + 31) // 32 * 4 + 255) // 256 * 256)
    rec = lib.proxtv_DR2L1W_TV_record_dev_f64
    o = torch.full_like(Yt, 3.0)
    t2 = torch.full((nb,), 7, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    bad = ((0, N, Yt, W1t, W2t, o, t2, nb), (M, 0, Yt, W1t, W2t, o, t2, nb), (M, N, None, W1t, W2t, o, t2, nb),
           (M, N, Yt, W1t, W2t, None, t2, nb), (M, N, Yt, W1t, W2t, o, None, nb), (M, N, Yt, None, W2t, o, t2, nb),
           (M, N, Yt, W1t, None, o, t2, nb), (M, N, Yt, W1t, W2t, o, t2, nb - 1))
    for i, (m, n, y, w1, w2, out, tp, sz) in enumerate(bad):
        info[:] = 0
        assert rec(m, n, _p(y), _p(w1), _p(w2), _p(out), K, _p(tp), sz, C.c_void_p(info.ctypes.data), None) == 0, i
        assert info[2] == 3, i
    # M == 1 needs no W1, N == 1 no W2
    y1 = torch.zeros((5, 1), dtype=torch.float64, device="cuda"); o1 = torch.empty_like(y1)
    t1 = torch.zeros(lib.proxtv_DR2L1W_TV_tape_bytes(1, 5, K), dtype=torch.uint8, device="cuda")
    assert rec(1, 5, _p(y1), None, _p(torch.ones(4, dtype=torch.float64, device="cuda")), _p(o1), K, _p(t1), t1.numel(), None, None) == 1
    assert rec(5, 1, _p(y1), _p(torch.ones(4, dtype=torch.float64, device="cuda")), None, _p(o1), K, _p(t1), t1.numel(), None, None) == 1
    # vjp refusals: shape, NULL arrays, another iteration count, dtype or shape, and a DR2_TV tape of the same image
    g = torch.randn_like(Yt)
    gY = torch.full_like(g, 3.0); gW1 = torch.full((N, M - 1), 3.0, dtype=torch.float64, device="cuda")
    gW2 = torch.full((N - 1, M), 3.0, dtype=torch.float64, device="cuda")
    vf = lib.proxtv_DR2L1W_TV_vjp_dev_f64
    for m, n, k in ((0, N, K), (M, 0, K), (M, N, K + 1), (M, N, 0), (M + 1, N, K), (N, M, K)):
        assert vf(m, n, k, _p(tape), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0, (m, n, k)
    assert vf(M, N, K, None, _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    assert vf(M, N, K, _p(tape), None, _p(gY), _p(gW1), _p(gW2), None) == 0
    assert vf(M, N, K, _p(tape), _p(g), None, _p(gW1), _p(gW2), None) == 0
    g32 = g.float(); gY32 = torch.full_like(g32, 3.0)
    assert lib.proxtv_DR2L1W_TV_vjp_dev_f32(M, N, K, _p(tape), _p(g32), _p(gY32), None, None, None) == 0     # recorded in float64
    dr2_tape = torch.zeros(lib.proxtv_DR2_TV_tape_bytes(M, N, 1, K), dtype=torch.uint8, device="cuda")
    o2 = torch.empty_like(Yt)
    assert lib.proxtv_DR2_TV_record_dev_f64(M, N, 1, 0, _p(Yt), 0.3, 0.3, _p(o2), K, _p(dr2_tape), dr2_tape.numel(), None, None) == 1
    assert vf(M, N, K, _p(dr2_tape), _p(g), _p(gY), _p(gW1), _p(gW2), None) == 0
    glam = torch.full((2,), 3.0, dtype=torch.float64, device="cuda")
    assert lib.proxtv_DR2_TV_vjp_dev_f64(M, N, 1, 0, K, _p(tape), _p(g), _p(gY), _p(glam), None) == 0          # and the converse
    torch.cuda.synchronize()
    assert bool((o == 3.0).all()) and bool((t2 == 7).all())
    assert all(bool((t == 3.0).all()) for t in (gY, gW1, gW2, gY32, glam))


# ---------------------------------------------------------------------------------------------------------------- autograd
def tensors(shape, seed, dt=torch.float64, zeros=0.0):
    Y, W1, W2 = problem(shape, seed, np.float64, zeros)
    rng = np.random.default_rng(seed)
    Y = Y + rng.normal(0, 1e-3, Y.shape)             # no ties
    return tuple(torch.tensor(a, dtype=dt, device="cuda") for a in (Y, W1, W2))


def test_gradcheck(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        x, w1, w2 = (t.requires_grad_(True) for t in tensors((6, 8), 21))
        assert torch.autograd.gradcheck(lambda a, b, c: ptv.tv1w_2d(a, b, c, max_iters=3), (x, w1, w2), eps=1e-6, atol=1e-6)
        x, w1, w2 = (t.requires_grad_(True) for t in tensors((5, 70), 22))          # the fast row route
        assert torch.autograd.gradcheck(lambda a, b, c: ptv.tv1w_2d(a, b, c, max_iters=2), (x, w1, w2), eps=1e-6, atol=1e-6)


def test_directional_differences(ptv):
    for shape in ((96, 130), (130, 40)):
        Y, W1, W2 = tensors(shape, 8, zeros=0.0)
        G = torch.randn(shape, dtype=torch.float64, device="cuda")
        fn = lambda a, b, c: ptv.tv1w_2d(a, b, c, max_iters=5)           # noqa: E731
        x, w1, w2 = (t.clone().requires_grad_(True) for t in (Y, W1, W2))
        (fn(x, w1, w2) * G).sum().backward()
        with torch.no_grad():
            base = fn(Y, W1, W2)
            for i, grad in enumerate((x.grad, w1.grad, w2.grad)):
                V = torch.randn_like(grad)

                def step(e):
                    args = [Y, W1, W2]
                    args[i] = args[i] + e * V
                    return ((fn(*args) - base) * G).sum().item()
                fd = kink_free_difference(step)
                an = (grad * V).sum().item()
                assert abs(fd - an) <= 2e-6 * max(abs(an), 1.0), (shape, i, fd, an)


def test_forward_equals_no_grad_and_each_input_alone(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            Y, W1, W2 = tensors((50, 90), 4, dt, zeros=0.2)
            G = torch.randn(Y.shape, dtype=dt, device="cuda")
            ref = ptv.tv1w_2d(Y, W1, W2)
            assert ref.grad_fn is None
            with torch.no_grad():
                assert ptv.tv1w_2d(Y.clone().requires_grad_(True), W1, W2).grad_fn is None
            full = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
            out = ptv.tv1w_2d(*full)
            assert out.grad_fn is not None and torch.equal(out.detach(), ref), (eng, dt)
            out.backward(G)
            for i in range(3):
                args = [Y, W1, W2]
                args[i] = args[i].clone().requires_grad_(True)
                o = ptv.tv1w_2d(*args)
                assert torch.equal(o.detach(), ref)
                o.backward(G)
                assert torch.equal(args[i].grad, full[i].grad), (eng, dt, i)


def test_mixed_dtypes_expanded_weights_and_views(ptv):
    M, N = 48, 80
    Y, W1, W2 = tensors((M, N), 6)
    G = torch.randn((M, N), dtype=torch.float64, device="cuda")
    # float32 image, float64 weights: the weight gradients come back in float64, equal to the float32 call's
    x = Y.float().requires_grad_(True)
    w1, w2 = W1.clone().requires_grad_(True), W2.clone().requires_grad_(True)
    ptv.tv1w_2d(x, w1, w2).backward(G.float())
    x32, a32, b32 = (t.float().requires_grad_(True) for t in (Y, W1, W2))
    ptv.tv1w_2d(x32, a32, b32).backward(G.float())
    assert w1.grad.dtype == torch.float64 and torch.equal(w1.grad, a32.grad.double()) and torch.equal(w2.grad, b32.grad.double())
    assert torch.equal(x.grad, x32.grad)
    # one learned scalar per axis through expand: the gradient is the sum of the per-edge maps
    s1 = torch.tensor(0.25, dtype=torch.float64, device="cuda", requires_grad=True)
    s2 = torch.tensor(0.4, dtype=torch.float64, device="cuda", requires_grad=True)
    ptv.tv1w_2d(Y, s1.expand(M - 1, N), s2.expand(M, N - 1)).backward(G)
    f1 = torch.full((M - 1, N), 0.25, dtype=torch.float64, device="cuda", requires_grad=True)
    f2 = torch.full((M, N - 1), 0.4, dtype=torch.float64, device="cuda", requires_grad=True)
    ptv.tv1w_2d(Y, f1, f2).backward(G)
    assert abs(s1.grad.item() - f1.grad.sum().item()) <= 1e-12 * max(abs(f1.grad).sum().item(), 1.0)
    assert abs(s2.grad.item() - f2.grad.sum().item()) <= 1e-12 * max(abs(f2.grad).sum().item(), 1.0)
    # non-contiguous x: a transposed view and a slice give the contiguous input's gradient
    xc = Y.clone().requires_grad_(True)
    ptv.tv1w_2d(xc, W1, W2).backward(G)
    for make in (lambda: Y.t().contiguous().t(), lambda: torch.nn.functional.pad(Y, (0, 3))[:, :N]):
        base = make().detach().requires_grad_(False)
        leaf = base.clone() if base.is_contiguous() else base
        leaf.requires_grad_(True)
        out = ptv.tv1w_2d(leaf, W1, W2)
        assert torch.equal(out.detach(), ptv.tv1w_2d(Y, W1, W2))
        out.backward(G)
        assert torch.equal(leaf.grad, xc.grad)


def test_non_default_stream(ptv, lib):
    Y, W1, W2 = tensors((64, 96), 2)
    G = torch.randn(Y.shape, dtype=torch.float64, device="cuda")
    a = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
    ptv.tv1w_2d(*a).backward(G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = [t.clone().requires_grad_(True) for t in (Y, W1, W2)]
        ptv.tv1w_2d(*b).backward(G)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, q.grad) for p, q in zip(a, b))
    # the C ABI on a non-default stream
    M, N = 64, 96
    Yt, W1t, W2t = colmajor(Y.cpu().numpy()), colmajor(W1.cpu().numpy()), colmajor(W2.cpu().numpy())
    g = torch.randn_like(Yt)
    out0, tape0 = record(lib, Yt, W1t, W2t, M, N, 3)
    r0 = vjp(lib, tape0, g, M, N, 3)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out1, tape1 = record(lib, Yt, W1t, W2t, M, N, 3, stream=s)
        r1 = vjp(lib, tape1, g, M, N, 3, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1) and torch.equal(tape0, tape1) and all(torch.equal(p, q) for p, q in zip(r0, r1))
