"""GPU tests (-m gpu) of the DR2_TV backward pass (DESIGN.md section 11): the segmentation tape, the tape-driven VJP kernels, the
recorded forward, the unrolled backward and the torch autograd path of tv1_2d / tv1_2d_batched.

Bars:
  * tape kernel == the numpy tape of the same y; tape-driven VJP == y-driven VJP (proxtv_prox_fibers_vjp_dev_*), bit for bit, over the
    shapes, cases and forced chunk lengths of test_gpu_vjp.py;
  * recorded forward == proxtv_DR2_TV_dev_* bit for bit on the lane schedules (both engines forced), <= 1e-6 relative on the chunked
    route; every recorded pass's tape == the host restatement's on dyadic inputs (test_gpu_lane.py's grid);
  * backward == the host restatement (dr2_vjp_emu.backward) to 1e-12 relative (float64) / 1e-5 (float32) -- the start value term and the
    penalty sums are the only sums whose order differs; two identical calls are bit-equal;
  * autograd: gradcheck, central differences, forward bit-equal to the no-grad call, layouts, streams, refusals.
"""
import ctypes as C

import numpy as np
import pytest

import dr2_vjp_emu as D
import lane_emu
import test_gpu_vjp as V
from conftest import relerr
from test_gpu_lane import dyadic
from vjp_emu import from_flat, to_flat

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

LAM = 0.375


@pytest.fixture(scope="module")
def emu():
    return lane_emu.load()


@pytest.fixture
def lib(ptv):
    L = ptv.load()
    L.proxtv_vjp_tuning(0)
    yield L
    L.proxtv_vjp_tuning(0)


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


def dev_tape(lib, y, nf, ln, inc, lam, w):
    nw = D.tape_words(nf * ln)
    F = torch.full((nw,), -1, dtype=torch.int32, device="cuda"); U = F.clone()
    f = lib.proxtv_fiber_tape_dev_f32 if y.dtype == torch.float32 else lib.proxtv_fiber_tape_dev_f64
    assert f(_p(y), nf, ln, inc, lam, _p(w), _p(F), _p(U), None) == 1, lib.proxtv_last_error()
    return F, U


def vjp_tape(lib, F, U, g, nf, ln, inc, want_gw):
    gx = torch.full_like(g, float("nan"))
    gw = torch.full((nf * max(ln - 1, 0),), float("nan"), dtype=g.dtype, device="cuda") if want_gw else None
    f = lib.proxtv_prox_fibers_vjp_tape_dev_f32 if g.dtype == torch.float32 else lib.proxtv_prox_fibers_vjp_tape_dev_f64
    assert f(_p(F), _p(U), _p(g), _p(gx), _p(gw), nf, ln, inc, None) == 1, lib.proxtv_last_error()
    return gx, gw


def as_u32(t):
    return t.cpu().numpy().view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- tape + tape-driven VJP
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_tape_and_tape_vjp_equal_y_driven(lib, dtype):
    rng = np.random.default_rng(0)
    for si, (nf, ln, inc) in enumerate(V.SHAPES):
        kind, lam, weighted = V.CASES[si % len(V.CASES)]
        if ln == 1_000_000:
            kind, lam, weighted = "blocks", 0.5, False
        x, y, g, w, Y, G, W, _, _ = V.run_case(lib, nf, ln, inc, kind, lam, weighted, dtype, rng)
        F, U = dev_tape(lib, y, nf, ln, inc, lam, w)
        Fn, Un = D.tape_bits(y.cpu().numpy(), nf, ln, inc, lam, W)
        assert np.array_equal(as_u32(F), Fn) and np.array_equal(as_u32(U), Un), (nf, ln, inc, kind, lam)
        for want in (True, False):
            gx0, gw0 = V.backward(lib, y, g, nf, ln, inc, lam, w, want)
            gx1, gw1 = vjp_tape(lib, F, U, g, nf, ln, inc, want)
            assert torch.equal(gx0, gx1), (nf, ln, inc, kind, lam, want)
            if want:
                assert torch.equal(gw0, gw1), (nf, ln, inc, kind, lam)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_tape_vjp_forced_chunk_lengths(lib, dtype):
    rng = np.random.default_rng(1)
    for (nf, ln, inc, kind, lam, weighted) in ((7, 3000, 1, "blocks", 0.3, False), (64, 2000, 32, "ties", 1.0, True),
                                                (1, 200_000, 1, "const", 0.5, False), (33, 1000, 3, "alt", 0.3, False)):
        x, y, g, w, Y, G, W, _, _ = V.run_case(lib, nf, ln, inc, kind, lam, weighted, dtype, rng)
        F, U = dev_tape(lib, y, nf, ln, inc, lam, w)
        for chunk in (1, 3, 32, 1000, 10 ** 7):
            lib.proxtv_vjp_tuning(chunk)
            gx0, gw0 = V.backward(lib, y, g, nf, ln, inc, lam, w, True)
            gx1, gw1 = vjp_tape(lib, F, U, g, nf, ln, inc, True)
            assert torch.equal(gx0, gx1) and torch.equal(gw0, gw1), (nf, ln, kind, chunk)


def test_tape_refusals_write_nothing(lib):
    y = torch.zeros(64, dtype=torch.float64, device="cuda")
    F = torch.full((64,), 7, dtype=torch.int32, device="cuda"); U = F.clone()
    for args in ((-1, 8, 1, 0.5), (8, -1, 1, 0.5), (8, 8, 0, 0.5), (6, 8, 4, 0.5), (8, 8, 1, -1.0)):
        assert lib.proxtv_fiber_tape_dev_f64(_p(y), *args, None, _p(F), _p(U), None) == 0, args
    assert lib.proxtv_fiber_tape_dev_f64(None, 8, 8, 1, 0.5, None, _p(F), _p(U), None) == 0
    gx = torch.full_like(y, 3.0)
    assert lib.proxtv_prox_fibers_vjp_tape_dev_f64(_p(F), None, _p(y), _p(gx), None, 8, 8, 1, None) == 0
    assert lib.proxtv_prox_fibers_vjp_tape_dev_f64(_p(F), _p(U), _p(y), _p(gx), None, 6, 8, 4, None) == 0
    torch.cuda.synchronize()
    assert bool((F == 7).all()) and bool((U == 7).all()) and bool((gx == 3.0).all())


# ---------------------------------------------------------------------------------------------------------------- recorded forward
def record(lib, Yt, M, N, batch, row_major, w1, w2, maxit, stream=None):
    """proxtv_DR2_TV_record_dev_*: (out, tape) for the device images Yt laid out as stated."""
    out = torch.full_like(Yt, float("nan"))
    nb = lib.proxtv_DR2_TV_tape_bytes(M, N, batch, maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    f = lib.proxtv_DR2_TV_record_dev_f32 if Yt.dtype == torch.float32 else lib.proxtv_DR2_TV_record_dev_f64
    assert f(M, N, batch, row_major, _p(Yt), w1, w2, _p(out), maxit, _p(tape), nb, C.c_void_p(info.ctypes.data), _st(stream)) == 1, \
        lib.proxtv_last_error()
    assert info[2] == 0
    return out, tape


def solve(lib, Yt, M, N, batch, row_major, w1, w2, maxit):
    out = torch.full_like(Yt, float("nan"))
    info = np.zeros(3)
    f = lib.proxtv_DR2_TV_dev_f32 if Yt.dtype == torch.float32 else lib.proxtv_DR2_TV_dev_f64
    f(M, N, batch, row_major, _p(Yt), w1, w2, _p(out), maxit, C.c_void_p(info.ctypes.data), _st())
    assert info[2] != 3, lib.proxtv_last_error()
    return out


def vjp(lib, tape, gout, M, N, batch, row_major, maxit, want_glam=True, stream=None):
    gY = torch.full_like(gout, float("nan"))
    glam = torch.full((2 * batch,), float("nan"), dtype=torch.float64, device="cuda") if want_glam else None
    f = lib.proxtv_DR2_TV_vjp_dev_f32 if gout.dtype == torch.float32 else lib.proxtv_DR2_TV_vjp_dev_f64
    assert f(M, N, batch, row_major, maxit, _p(tape), _p(gout), _p(gY), _p(glam), _st(stream)) == 1, lib.proxtv_last_error()
    return gY, glam


def device_images(Y, row_major, dt):
    """Y (B, M, N) numpy -> device tensor in the stated storage order (column-major: each image's transpose, C-ordered)."""
    T = torch.float64 if dt == np.float64 else torch.float32
    return torch.tensor(Y if row_major else np.ascontiguousarray(Y.transpose(0, 2, 1)), dtype=T, device="cuda")


def host_images(t, row_major):
    a = t.cpu().numpy()
    return a if row_major else np.ascontiguousarray(a.transpose(0, 2, 1))


def pass_tapes(tape, n, K):
    sb = D.tape_words(n) * 4
    raw = tape.cpu().numpy()[256:].view(np.uint32).reshape(2 * K + 1, 2, sb // 4)
    return raw


@pytest.mark.parametrize("maxit", [1, 2, 35])
@pytest.mark.parametrize("shape", [(52, 36), (100, 140)], ids=["52x36", "100x140"])
def test_recorded_forward_and_backward_on_lane_schedules(lib, engine, emu, shape, maxit):
    """Dyadic images, both lane engines, both storage orders, batch 1 and 3, float64 and float32: out == proxtv_DR2_TV_dev_* and ==
    the host restatement bit for bit, every pass's tape == the restatement's, and the backward == the restatement."""
    M, N = shape
    it_arg = 0 if maxit == 35 else maxit
    w1, w2 = LAM, 0.25
    for dt in (np.float64, np.float32):
        for batch in (1, 3):
            Y = dyadic((batch, M, N), 7 * batch, dt)
            want, passes = D.forward(emu, Y, w1, w2, maxit)
            G = np.random.default_rng(batch).normal(size=Y.shape).astype(dt)
            gY_h, glam_h = D.backward(passes, G, w1, w2, maxit)
            for eng in ("lane", "lane-t"):
                engine(eng)
                for row_major in (1, 0):
                    what = (shape, maxit, np.dtype(dt).name, batch, eng, row_major)
                    Yt = device_images(Y, row_major, dt)
                    out, tape = record(lib, Yt, M, N, batch, row_major, w1, w2, it_arg)
                    assert torch.equal(out, solve(lib, Yt, M, N, batch, row_major, w1, w2, it_arg)), what
                    assert np.array_equal(host_images(out, row_major), want), what
                    raw = pass_tapes(tape, batch * M * N, maxit)
                    for p, X in enumerate(passes):
                        col = p % 2 == 1
                        Xs = X if row_major else np.ascontiguousarray(X.transpose(0, 2, 1))
                        if row_major:
                            geo = (batch * N, M, N) if col else (batch * M, N, 1)
                        else:
                            geo = (batch * N, M, 1) if col else (batch * M, N, M)
                        Fn, Un = D.tape_bits(Xs, *geo, w1 if col else w2)
                        assert np.array_equal(raw[p, 0], Fn) and np.array_equal(raw[p, 1], Un), what + (p,)
                    gY, glam = vjp(lib, tape, device_images(G, row_major, dt), M, N, batch, row_major, it_arg)
                    tol = 1e-12 if dt == np.float64 else 1e-5
                    assert relerr(host_images(gY, row_major), gY_h) <= tol, what
                    assert relerr(glam.cpu().numpy().reshape(batch, 2), glam_h) <= tol, what


def test_recorded_forward_4096_and_chunked_route(lib, engine):
    """4096 x 4096 float64 on the lane schedules (bit for bit), and lambda above the lane guard (chunked engine) within 1e-6."""
    M = N = 4096
    rng = np.random.default_rng(3)
    Y = dyadic((1, M, N), 5, np.float64)
    Yt = torch.tensor(Y[0], device="cuda")
    for eng in ("lane", "lane-t"):
        engine(eng)
        out, tape = record(lib, Yt, M, N, 1, 1, LAM, LAM, 0)
        assert torch.equal(out, solve(lib, Yt, M, N, 1, 1, LAM, LAM, 0)), eng
        del tape
    engine("auto")
    Z = torch.tensor(rng.normal(size=(512, 384)), device="cuda")
    for row_major, Zt in ((1, Z), (0, Z.t().contiguous())):
        Ms, Ns = (512, 384)
        out, _ = record(lib, Zt, Ms, Ns, 1, row_major, 5.0, 5.0, 0)
        assert lib.proxtv_lane_guard_last() == 0
        ref = solve(lib, Zt, Ms, Ns, 1, row_major, 5.0, 5.0, 0)
        assert relerr(out.cpu().numpy(), ref.cpu().numpy()) <= 1e-6, row_major


def test_backward_deterministic_and_refusals(lib, emu):
    M, N, batch = 64, 48, 2
    Y = dyadic((batch, M, N), 9, np.float64)
    Yt = device_images(Y, 1, np.float64)
    out, tape = record(lib, Yt, M, N, batch, 1, 0.3, 0.2, 5)
    g = torch.randn_like(Yt)
    a = vjp(lib, tape, g, M, N, batch, 1, 5)
    b = vjp(lib, tape, g, M, N, batch, 1, 5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    gY0, _ = vjp(lib, tape, g, M, N, batch, 1, 5, want_glam=False)
    assert torch.equal(gY0, a[0])
    # refusals leave the outputs untouched
    gY = torch.full_like(g, 3.0); glam = torch.full((2 * batch,), 3.0, dtype=torch.float64, device="cuda")
    f = lib.proxtv_DR2_TV_vjp_dev_f64
    for args in ((M, N, batch, 1, 6), (M, N + 1, batch, 1, 5), (M, N, batch, 0, 5), (M, N, 1, 1, 5), (0, N, batch, 1, 5),
                 (M, N, 0, 1, 5)):
        assert f(*args, _p(tape), _p(g), _p(gY), _p(glam), None) == 0, args
    assert f(M, N, batch, 1, 5, None, _p(g), _p(gY), _p(glam), None) == 0
    assert f(M, N, batch, 1, 5, _p(tape), _p(g), None, _p(glam), None) == 0
    g32 = g.float(); gY32 = torch.full_like(g32, 3.0)
    assert lib.proxtv_DR2_TV_vjp_dev_f32(M, N, batch, 1, 5, _p(tape), _p(g32), _p(gY32), None, None) == 0      # recorded in float64
    torch.cuda.synchronize()
    assert bool((gY == 3.0).all()) and bool((glam == 3.0).all()) and bool((gY32 == 3.0).all())
    # record refusals: short tape, bad shape, NULL arrays, negative weight
    o = torch.full_like(Yt, 3.0); small = torch.full((1024,), 7, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    rec = lib.proxtv_DR2_TV_record_dev_f64
    nb = lib.proxtv_DR2_TV_tape_bytes(M, N, batch, 5)
    assert nb == 256 + 11 * 2 * D.tape_words(M * N * batch) * 4
    assert rec(M, N, batch, 1, _p(Yt), 0.3, 0.2, _p(o), 5, _p(small), 1024, C.c_void_p(info.ctypes.data), None) == 0 and info[2] == 3
    assert rec(M, N, 0, 1, _p(Yt), 0.3, 0.2, _p(o), 5, _p(tape), nb, None, None) == 0
    assert rec(M, N, batch, 1, _p(Yt), -0.3, 0.2, _p(o), 5, _p(tape), nb, None, None) == 0
    assert rec(M, N, batch, 1, None, 0.3, 0.2, _p(o), 5, _p(tape), nb, None, None) == 0
    torch.cuda.synchronize()
    assert bool((o == 3.0).all()) and bool((small == 7).all())
    assert lib.proxtv_DR2_TV_tape_bytes(4096, 4096, 1, 35) == 256 + 71 * 2 * (4096 * 4096 // 32 * 4)


# ---------------------------------------------------------------------------------------------------------------- autograd
def test_gradcheck(ptv, engine):
    rng = np.random.default_rng(21)
    for eng in ("auto", "lane"):
        engine(eng)
        x = torch.tensor(rng.normal(size=(8, 12)), device="cuda", requires_grad=True)
        assert torch.autograd.gradcheck(lambda a: ptv.tv1_2d(a, 0.3, max_iters=4), (x,), eps=1e-6, atol=1e-6)
        xb = torch.tensor(rng.normal(size=(2, 6, 8)), device="cuda", requires_grad=True)
        assert torch.autograd.gradcheck(lambda a: ptv.tv1_2d_batched(a, 0.25, max_iters=3), (xb,), eps=1e-6, atol=1e-6)
        w = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
        xc = x.detach()
        assert torch.autograd.gradcheck(lambda ww: ptv.tv1_2d(xc, ww, max_iters=4), (w,), eps=1e-6, atol=1e-6)
        assert torch.autograd.gradcheck(lambda a, ww: ptv.tv1_2d_batched(a, ww), (xb, w), eps=1e-6, atol=1e-6)


FD_TOL = 2e-6


def kink_free_difference(f, eps_list=(1e-6, 3e-7, 1e-7, 3e-8, 1e-8)):
    """Central difference of a piecewise linear function of one step size (f(e) -> the change of the objective, formed as a sum of
    elementwise output differences) at the first step whose two one-sided differences agree to FD_TOL, i.e. no segment merges or
    splits inside it that changes the slope by more than that (with 71 passes over 10^5 edges each, a step of 1e-6 often contains
    such a kink; below 1e-8 rounding takes over)."""
    for eps in eps_list:
        p, m = f(eps) / eps, -f(-eps) / eps
        if abs(p - m) <= FD_TOL * max(abs(p), abs(m)):
            return (p + m) / 2
    raise AssertionError("every step crosses a kink")


def test_directional_differences_on_lane_route(ptv):
    """5 iterations: the unrolled solve is a composition of piecewise linear maps whose pieces multiply with every pass; at 35
    iterations on 2 x 256 x 384 no step between 1e-8 and 1e-6 is free of kinks for every image (35 iterations are covered by the
    restatement comparison and gradcheck above)."""
    rng = np.random.default_rng(8)
    for shape, fn0 in (((256, 384), ptv.tv1_2d), ((2, 256, 384), ptv.tv1_2d_batched)):
        fn = lambda a, ww, f=fn0: f(a, ww, max_iters=5)           # noqa: E731
        Y = torch.tensor(rng.normal(size=shape), device="cuda")
        G = torch.tensor(rng.normal(size=shape), device="cuda")
        x = Y.clone().requires_grad_(True)
        w = torch.tensor(0.2, dtype=torch.float64, device="cuda", requires_grad=True)
        (fn(x, w) * G).sum().backward()
        assert ptv.load().proxtv_lane_guard_last() == 1
        Vd = torch.tensor(rng.normal(size=shape), device="cuda")
        with torch.no_grad():
            base = fn(Y, 0.2)
            fd = kink_free_difference(lambda e: ((fn(Y + e * Vd, 0.2) - base) * G).sum().item())
            fdw = kink_free_difference(lambda e: ((fn(Y, 0.2 + e) - base) * G).sum().item())
        an = (x.grad * Vd).sum().item()
        assert abs(fd - an) <= FD_TOL * max(abs(an), 1.0), (shape, fd, an)
        assert abs(fdw - w.grad.item()) <= FD_TOL * max(abs(fdw), 1.0), (shape, fdw, w.grad.item())


def test_autograd_forward_equals_no_grad_and_layouts(ptv, lib, engine):
    rng = np.random.default_rng(12)
    Y = dyadic((3, 52, 36), 4, np.float64)[0]
    for dt in (torch.float64, torch.float32):
        base = torch.tensor(Y, dtype=dt, device="cuda")
        views = (base,                                                         # row-major
                 torch.tensor(np.ascontiguousarray(Y.T), dtype=dt, device="cuda").t(),   # column-major view
                 torch.tensor(np.ascontiguousarray(np.pad(Y, ((0, 0), (0, 4)))), dtype=dt, device="cuda")[:, :36])  # copied
        for eng in ("auto", "lane", "lane-t"):
            engine(eng)
            for v in views:
                ref = ptv.tv1_2d(v, 0.2)
                assert ref.grad_fn is None
                x = v.detach().clone() if v.is_contiguous() else v.detach()
                x.requires_grad_(True)
                out = ptv.tv1_2d(x, 0.2)
                assert lib.proxtv_lane_guard_last() != 0 or eng != "auto"
                assert out.grad_fn is not None and torch.equal(out.detach(), ref), (dt, eng, v.stride())
                G = torch.tensor(rng.normal(size=Y.shape), dtype=dt, device="cuda")
                out.backward(G)
                assert x.grad.shape == x.shape and torch.isfinite(x.grad).all()
        # the same gradient whatever the layout of the upstream gradient
        x = base.clone().requires_grad_(True)
        out = ptv.tv1_2d(x, LAM)
        G = torch.tensor(rng.normal(size=Y.shape), dtype=dt, device="cuda")
        g1, = torch.autograd.grad(out, x, G, retain_graph=True)
        g2, = torch.autograd.grad(out, x, G.t().contiguous().t())
        assert torch.equal(g1, g2)
    x = torch.tensor(Y, device="cuda")
    assert ptv.tv1_2d(x, LAM).grad_fn is None
    with torch.no_grad():
        assert ptv.tv1_2d(x.clone().requires_grad_(True), LAM).grad_fn is None


def test_autograd_non_default_stream(ptv):
    rng = np.random.default_rng(2)
    Y = torch.tensor(rng.normal(size=(2, 64, 96)), device="cuda")
    G = torch.tensor(rng.normal(size=(2, 64, 96)), device="cuda")
    x0 = Y.clone().requires_grad_(True)
    ptv.tv1_2d_batched(x0, 0.3).backward(G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        x1 = Y.clone().requires_grad_(True)
        ptv.tv1_2d_batched(x1, 0.3).backward(G)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(x0.grad, x1.grad)


def test_record_and_backward_on_a_stream(lib):
    """The C ABI on a non-default stream equals the default stream's results."""
    M, N = 64, 80
    Y = dyadic((1, M, N), 3, np.float32)
    Yt = device_images(Y, 0, np.float32)
    g = torch.randn_like(Yt)
    out0, tape0 = record(lib, Yt, M, N, 1, 0, 0.3, 0.3, 3)
    gY0, gl0 = vjp(lib, tape0, g, M, N, 1, 0, 3)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out1, tape1 = record(lib, Yt, M, N, 1, 0, 0.3, 0.3, 3, stream=s)
        gY1, gl1 = vjp(lib, tape1, g, M, N, 1, 0, 3, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1) and torch.equal(tape0, tape1) and torch.equal(gY0, gY1) and torch.equal(gl0, gl1)
