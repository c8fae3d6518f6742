"""GPU tests (-m gpu) of the PDR_TV backward pass (DESIGN.md section 13): the recorded forward, the unrolled backward and the torch
autograd path of tvgen_pdr.

Bars:
  * recorded forward == proxtv_PDR_TV_dev_* bit for bit, x and info, on the engines seq, chunked, lane and auto, float64 and float32,
    1D to 4D, 1 to 5 terms (both combine kernels; a misaligned output forces the generic one), 1 / 2 / 35 iterations, and the
    512 x 512 x 256 float32 volume with 3 terms; in float64 every recorded pass's tape == the host forward's (pdr_vjp_emu.forward:
    the oracle's exact prox under seq / chunked, lane_emu.slope_fibers on the lane route);
  * backward == the host restatement driven by the device's own tape (pdr_vjp_emu.backward_from_tapes): gY bit for bit (float64 and
    float32), glam to 1e-12 relative (its sums are the only order-dependent ones); two identical calls are bit-equal and a NULL glam
    leaves gY unchanged;
  * refusals write nothing (lambdas included); autograd: gradcheck, directional differences, forward bit-equal to the no-grad call,
    layouts and views, ws as a list / ndarray / tensor and never modified, a batch axis without a term, a non-default stream.
"""
import ctypes as C

import numpy as np
import pytest

import lane_emu
import pdr_vjp_emu as P
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


def _a(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _st(stream=None):
    return C.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)


def tdt(dt):
    return torch.float32 if dt == np.float32 else torch.float64


def flat_buffer(y, dt, misaligned=False):
    """The flat column-major array y on the device; misaligned: a view one element into a larger buffer (not 16-byte aligned)."""
    t = torch.tensor(np.concatenate([[0.0], y]) if misaligned else y, dtype=tdt(dt), device="cuda")
    return t[1:] if misaligned else t


def like(t, value, misaligned=False):
    buf = torch.full((t.numel() + (1 if misaligned else 0),), value, dtype=t.dtype, device="cuda")
    return buf[1:] if misaligned else buf


def record(lib, yt, ns, ws, ds, maxit, misaligned=False, stream=None):
    nsa, dsa, lam = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64), np.array(ws, dtype=np.float64)
    nb = lib.proxtv_PDR_TV_tape_bytes(_a(nsa), len(ns), len(ws), maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    out = like(yt, float("nan"), misaligned)
    info = np.zeros(3)
    f = lib.proxtv_PDR_TV_record_dev_f32 if yt.dtype == torch.float32 else lib.proxtv_PDR_TV_record_dev_f64
    assert f(_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _p(tape), nb, _st(stream)) == 1, \
        lib.proxtv_last_error()
    assert np.array_equal(lam, np.array(ws, dtype=np.float64) * len(ws))               # scaled in place like the no-grad call
    return out, tape, info


def solve(lib, yt, ns, ws, ds, maxit, misaligned=False):
    nsa, dsa, lam = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64), np.array(ws, dtype=np.float64)
    out = like(yt, float("nan"), misaligned)
    info = np.zeros(3)
    f = lib.proxtv_PDR_TV_dev_f32 if yt.dtype == torch.float32 else lib.proxtv_PDR_TV_dev_f64
    assert f(_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _st()) == 1, lib.proxtv_last_error()
    return out, info


def vjp(lib, tape, gout, ns, ds, maxit, want_glam=True, stream=None):
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    gY = torch.full_like(gout, float("nan"))
    glam = torch.full((len(ds),), float("nan"), dtype=torch.float64, device="cuda") if want_glam else None
    f = lib.proxtv_PDR_TV_vjp_dev_f32 if gout.dtype == torch.float32 else lib.proxtv_PDR_TV_vjp_dev_f64
    assert f(_a(nsa), len(ns), len(ds), _a(dsa), maxit, _p(tape), _p(gout), _p(gY), _p(glam), _st(stream)) == 1, lib.proxtv_last_error()
    return gY, glam


def check_backward(lib, tape, G, ns, ds, maxit, what):
    """Device backward against the restatement driven by the device's own tape."""
    K = maxit if maxit > 0 else P.MAX_ITERS
    n = G.size
    gY, glam = vjp(lib, tape, torch.tensor(G, device="cuda"), ns, ds, maxit)
    hY, hlam = P.backward_from_tapes(P.device_pass_tapes(tape.cpu().numpy(), n, len(ds), K), G, ns, ds, K)
    assert np.array_equal(gY.cpu().numpy(), hY), what
    g = glam.cpu().numpy()
    assert np.abs(g - hlam).max() <= 1e-12 * max(np.abs(hlam).max(), 1e-300), what


# (ns, ws, ds): 1D to 4D, 1 to 5 terms, a repeated axis, a zero penalty, an axis without a term, a length-1 axis
CASES = [((3000,), [0.4], [1]),
         ((96, 80), [0.3, 0.2], [1, 2]),
         ((40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3]),
         ((12, 10, 8, 6), [0.3, 0.1, 0.2, 0.4], [1, 2, 3, 4]),
         ((20, 18, 16), [0.2, 0.1, 0.3, 0.15, 0.0], [1, 2, 3, 1, 2]),
         ((30, 1, 70), [0.3, 0.2], [3, 2])]


def case_input(ns, seed, dt):
    return dyadic((1, int(np.prod(ns)) // ns[-1], ns[-1]), seed, np.float64).ravel().astype(dt)


@pytest.mark.parametrize("maxit", [1, 2, 35])
def test_recorded_forward_equals_solve_and_backward(lib, engine, maxit):
    it_arg = 0 if maxit == 35 else maxit
    for ci, (ns, ws, ds) in enumerate(CASES):
        for dt in (np.float64, np.float32):
            y = case_input(ns, 3 + ci, dt)
            yt = flat_buffer(y, dt)
            G = np.random.default_rng(ci).normal(size=y.size).astype(dt)
            for eng in ("seq", "chunked", "lane", "auto"):
                engine(eng)
                for mis in ((False, True) if eng == "auto" else (False,)):
                    what = (ns, len(ws), maxit, np.dtype(dt).name, eng, mis)
                    out, tape, info = record(lib, yt, ns, ws, ds, it_arg, misaligned=mis)
                    ref, rinfo = solve(lib, yt, ns, ws, ds, it_arg, misaligned=mis)
                    assert torch.equal(out, ref) and np.array_equal(info, rinfo), what
                    if eng in ("seq", "auto") and not mis:
                        check_backward(lib, tape, G, ns, ds, it_arg, what)


@pytest.mark.parametrize("maxit", [2, 35])
def test_tapes_equal_host_forward(lib, engine, port, maxit):
    """float64: under seq / chunked every pass is the exact prox; on the lane route (every axis >= 64 long, >= 1024 fibers) the
    slope-form scan.  The recorded output equals the host forward's and the no-grad solve's."""
    it_arg = 0 if maxit == 35 else maxit
    exact = P.exact_prox(port)
    emu = lane_emu.load()
    slope = P.slope_prox(emu)

    def lane_route(a, nf, ln, inc, lam):
        return (slope if lam > 0 and ln >= 64 and nf >= 1024 else exact)(a, nf, ln, inc, lam)
    for ns, ws, ds, engines in (((40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3], ("seq", "chunked")),
                                ((20, 18, 16), [0.2, 0.1, 0.3, 0.15, 0.0], [1, 2, 3, 1, 2], ("seq", "chunked")),
                                ((96, 80), [0.3, 0.2], [2, 1], ("seq", "chunked")),
                                ((64, 64, 64), [0.15, 0.2, 0.25], [1, 2, 3], ("lane",))):
        y = case_input(ns, 7, np.float64)
        yt = flat_buffer(y, np.float64)
        for eng in engines:
            engine(eng)
            want, passes = P.forward(lane_route if eng == "lane" else exact, y, ns, ws, ds, maxit)
            host = P.pass_tapes(passes, ns, ws, ds)
            out, tape, info = record(lib, yt, ns, ws, ds, it_arg)
            assert np.array_equal(out.cpu().numpy(), want), (ns, eng)
            ref, rinfo = solve(lib, yt, ns, ws, ds, it_arg)
            assert torch.equal(out, ref) and np.array_equal(info, rinfo), (ns, eng)
            dev = P.device_pass_tapes(tape.cpu().numpy(), y.size, len(ws), maxit)
            assert len(dev) == len(host) == (maxit - 1) * len(ws)
            for p, ((F, U), (Fh, Uh)) in enumerate(zip(dev, host)):
                assert np.array_equal(F, Fh) and np.array_equal(U, Uh), (ns, eng, p)


def test_volume_512(lib, engine):
    """512 x 512 x 256 float32, 3 terms (BASELINE config 4's volume): the recorded forward equals the solve."""
    import synth_inputs as S
    ns, ws, ds = (512, 512, 256), [0.2, 0.2, 0.2], [1, 2, 3]
    yt = torch.from_numpy(np.ascontiguousarray(S.gen_cfg4(ns, seed=0).ravel(order="F"))).to(device="cuda", dtype=torch.float32)
    engine("auto")
    out, tape, info = record(lib, yt, ns, ws, ds, 0)
    ref, rinfo = solve(lib, yt, ns, ws, ds, 0)
    assert torch.equal(out, ref) and np.array_equal(info, rinfo)
    assert tape.numel() == 256 + 34 * 3 * 2 * (512 * 512 * 256 // 32 * 4)


def test_backward_deterministic_and_null_glam(lib):
    ns, ws, ds = (48, 40, 24), [0.2, 0.3, 0.25], [1, 2, 3]
    y = case_input(ns, 9, np.float64)
    _, tape, _ = record(lib, flat_buffer(y, np.float64), ns, ws, ds, 5)
    g = torch.randn(y.size, dtype=torch.float64, device="cuda")
    a = vjp(lib, tape, g, ns, ds, 5)
    b = vjp(lib, tape, g, ns, ds, 5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(vjp(lib, tape, g, ns, ds, 5, want_glam=False)[0], a[0])


def test_refusals_write_nothing(lib):
    ns, ws, ds, K = (20, 16, 12), [0.2, 0.3, 0.1], [1, 2, 3], 3
    y = case_input(ns, 2, np.float64)
    yt = flat_buffer(y, np.float64)
    _, tape, _ = record(lib, yt, ns, ws, ds, K)
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    nb = lib.proxtv_PDR_TV_tape_bytes(_a(nsa), 3, 3, K)
    assert nb == 256 + (K - 1) * 3 * 2 * (((y.size + 31) // 32 * 4 + 255) // 256 * 256)
    rec = lib.proxtv_PDR_TV_record_dev_f64
    o = torch.full_like(yt, 3.0)
    t2 = torch.full((nb,), 7, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    lam0 = np.array(ws)
    big = np.arange(1, 66, dtype=np.float64) % 3 + 1
    lam65 = np.full(65, 0.1)
    bad = [dict(y=None), dict(x=None), dict(lam=None), dict(dims=None), dict(ns=None), dict(tape=None),
           dict(nds=0), dict(nds=17), dict(ns=np.array([20, -16, 12], dtype=np.int32)), dict(npen=0),
           dict(npen=65, lam=lam65, dims=big), dict(dims=np.array([1.0, 2.0, 4.0])), dict(dims=np.array([0.0, 2.0, 3.0])),
           dict(lam=np.array([0.2, -0.3, 0.1])), dict(tb=nb - 1)]
    for i, kw in enumerate(bad):
        lam = kw.get("lam", lam0).copy() if kw.get("lam", lam0) is not None else None
        nsx = kw.get("ns", nsa)
        nds = kw.get("nds", 3)
        nsx17 = np.full(17, 1, dtype=np.int32) if nds == 17 else nsx
        info[:] = 0
        r = rec(_p(kw.get("y", yt)), _a(lam), _a(kw.get("dims", dsa)), _p(kw.get("x", o)), _a(info), _a(nsx17), nds,
                kw.get("npen", 3), K, _p(kw.get("tape", t2)), kw.get("tb", nb), None)
        assert r == 0 and info[2] == 3, i
        if lam is not None:
            assert np.array_equal(lam, kw.get("lam", lam0)), i                  # not scaled
    # vjp refusals: NULL arrays, another iteration count, dtype, shape, axes or term count, and the tapes of DR2_TV / DR2L1W_TV
    g = torch.randn_like(yt)
    gY = torch.full_like(g, 3.0)
    glam = torch.full((3,), 3.0, dtype=torch.float64, device="cuda")
    vf = lib.proxtv_PDR_TV_vjp_dev_f64

    def call(f=vf, nsx=nsa, nds=3, npen=3, dims=dsa, k=K, tp=tape, gg=g, gy=gY):
        return f(_a(nsx), nds, npen, _a(dims), k, _p(tp), _p(gg), _p(gy), _p(glam), None)
    assert call(k=K + 1) == 0 and call(k=0) == 0
    assert call(nsx=np.array([20, 12, 16], dtype=np.int32)) == 0
    assert call(dims=np.array([1.0, 3.0, 2.0])) == 0
    assert call(npen=2) == 0 and call(nds=2) == 0
    assert call(tp=None) == 0 and call(gg=None) == 0 and call(gy=None) == 0
    g32 = g.float(); gY32 = torch.full_like(g32, 3.0)
    assert call(f=lib.proxtv_PDR_TV_vjp_dev_f32, gg=g32, gy=gY32) == 0                    # recorded in float64
    M, N = 20, 192                                                                      # the same number of elements as an image
    dr2 = torch.zeros(lib.proxtv_DR2_TV_tape_bytes(M, N, 1, K), dtype=torch.uint8, device="cuda")
    o2 = torch.empty_like(yt)
    assert lib.proxtv_DR2_TV_record_dev_f64(M, N, 1, 0, _p(yt), 0.3, 0.3, _p(o2), K, _p(dr2), dr2.numel(), None, None) == 1
    drw = torch.zeros(lib.proxtv_DR2L1W_TV_tape_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    w1 = torch.full(((M - 1) * N,), 0.2, dtype=torch.float64, device="cuda")
    w2 = torch.full((M * (N - 1),), 0.2, dtype=torch.float64, device="cuda")
    assert lib.proxtv_DR2L1W_TV_record_dev_f64(M, N, _p(yt), _p(w1), _p(w2), _p(o2), K, _p(drw), drw.numel(), None, None) == 1
    for other in (dr2, drw):
        big_enough = torch.zeros(max(other.numel(), nb), dtype=torch.uint8, device="cuda")
        big_enough[:other.numel()] = other
        assert call(tp=big_enough) == 0
    torch.cuda.synchronize()
    assert bool((o == 3.0).all()) and bool((t2 == 7).all())
    assert bool((gY == 3.0).all()) and bool((glam == 3.0).all()) and bool((gY32 == 3.0).all())


# ---------------------------------------------------------------------------------------------------------------- autograd
def volume(shape, seed, dt=torch.float64):
    rng = np.random.default_rng(seed)
    return torch.tensor(rng.normal(size=shape), dtype=dt, device="cuda")


def test_gradcheck(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        x = volume((6, 5, 4), 21).requires_grad_(True)
        w = torch.tensor([0.2, 0.3, 0.25], dtype=torch.float64, device="cuda", requires_grad=True)
        assert torch.autograd.gradcheck(lambda a, b: ptv.tvgen_pdr(a, b, [1, 2, 3], [1, 1, 1], max_iters=3), (x, w), eps=1e-6, atol=1e-6)
        x2 = volume((9, 7), 22).requires_grad_(True)
        assert torch.autograd.gradcheck(lambda a: ptv.tvgen_pdr(a, [0.3, 0.2], [1, 2], [1, 1], max_iters=4), (x2,), eps=1e-6, atol=1e-6)


def test_directional_differences(ptv):
    """A few iterations on noise: the unrolled map's linear pieces multiply with every pass, and at many iterations or on larger
    arrays no step between 1e-8 and 1e-6 is free of kinks (35 iterations are covered by the restatement comparison above)."""
    for shape, ws, ds, K in (((40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3], 5), ((96, 64), [0.3, 0.2], [1, 2], 4)):
        Y = volume(shape, 8)
        G = volume(shape, 9)
        x = Y.clone().requires_grad_(True)
        w = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
        fn = lambda a, b, ds=ds, K=K: ptv.tvgen_pdr(a, b, ds, [1] * len(ds), max_iters=K)           # noqa: E731
        (fn(x, w) * G).sum().backward()
        with torch.no_grad():
            base = fn(Y, ws)
            V = volume(shape, 10)
            fd = kink_free_difference(lambda e: ((fn(Y + e * V, ws) - base) * G).sum().item())
            an = (x.grad * V).sum().item()
            assert abs(fd - an) <= 2e-6 * max(abs(an), 1.0), (shape, fd, an)
            for i in range(len(ws)):
                def step(e):
                    wh = list(ws); wh[i] += e
                    return ((fn(Y, wh) - base) * G).sum().item()
                fdw = kink_free_difference(step)
                assert abs(fdw - w.grad[i].item()) <= 2e-6 * max(abs(fdw), 1.0), (shape, i, fdw, w.grad[i].item())


def test_forward_equals_no_grad_layouts_and_ws(ptv, engine):
    """C order, Fortran order and a non-contiguous view; ws as a list, an ndarray and tensors of two dtypes and devices (never
    modified); the result keeps x's memory order.  The penalties are exact in float32, so every form of ws carries the same values."""
    ws, ds = [0.25, 0.375, 0.125], [1, 2, 3]
    for eng in ("seq", "auto"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            Y = volume((24, 20, 16), 4, dt)
            G = volume((24, 20, 16), 5, dt)
            ref = ptv.tvgen_pdr(Y, ws, ds, [1, 1, 1])
            assert ref.grad_fn is None and ref.is_contiguous() and ptv.tvgen_pdr.last_info[0] == 35
            grads = []
            for make in (lambda: Y.clone(), lambda: Y.permute(2, 1, 0).contiguous().permute(2, 1, 0),
                         lambda: torch.nn.functional.pad(Y, (0, 3))[:, :, :16]):
                v = make()
                no_grad = ptv.tvgen_pdr(v, ws, ds, [1, 1, 1])
                x = v.detach().requires_grad_(True)
                out = ptv.tvgen_pdr(x, ws, ds, [1, 1, 1])
                assert out.grad_fn is not None and torch.equal(out.detach(), no_grad), (eng, dt)
                if eng == "seq":
                    assert torch.equal(no_grad, ref), (eng, dt, v.stride())
                else:
                    assert float((no_grad - ref).abs().max()) <= (1e-12 if dt == torch.float64 else 1e-5) * float(ref.abs().max())
                assert out.stride() == (v.stride() if (v.is_contiguous() or ptv._f_contiguous(v)) else ref.stride())
                out.backward(G)
                grads.append(x.grad)
            if eng == "seq":
                assert all(torch.equal(g, grads[0]) for g in grads)
            with torch.no_grad():
                assert ptv.tvgen_pdr(Y.clone().requires_grad_(True), ws, ds, [1, 1, 1]).grad_fn is None
            # ws: list / ndarray / tensors -- same result, same x gradient, ws untouched
            wl, wa = list(ws), np.array(ws)
            wt64 = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
            wt32 = torch.tensor(ws, dtype=torch.float32, requires_grad=True)                  # float32 on the CPU
            res = []
            for w in (wl, wa, wt64, wt32):
                x = Y.clone().requires_grad_(True)
                out = ptv.tvgen_pdr(x, w, ds, [1, 1, 1])
                out.backward(G)
                res.append((out.detach(), x.grad))
            assert all(torch.equal(r[0], res[0][0]) and torch.equal(r[1], res[0][1]) for r in res)
            assert wl == ws and np.array_equal(wa, ws) and torch.equal(wt64.detach().cpu(), torch.tensor(ws, dtype=torch.float64))
            assert wt32.grad.dtype == torch.float32 and wt32.grad.device.type == "cpu"
            assert torch.equal(wt32.grad, wt64.grad.cpu().float())                         # the same float64 gradient, cast


def test_batch_axis_equals_slices(ptv, engine):
    """A leading batch axis without a term: bit for bit the per-slice solves and gradients."""
    for eng in ("seq", "chunked"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            X = volume((3, 40, 72), 6, dt)
            G = volume((3, 40, 72), 7, dt)
            x = X.clone().requires_grad_(True)
            out = ptv.tvgen_pdr(x, [0.3, 0.2], [2, 3], [1, 1], max_iters=6)
            out.backward(G)
            for b in range(3):
                xb = X[b].clone().requires_grad_(True)
                ob = ptv.tvgen_pdr(xb, [0.3, 0.2], [1, 2], [1, 1], max_iters=6)
                ob.backward(G[b])
                assert torch.equal(ob.detach(), out.detach()[b]) and torch.equal(xb.grad, x.grad[b]), (eng, dt, b)


def test_non_default_stream(ptv, lib):
    Y, G = volume((32, 24, 16), 2), volume((32, 24, 16), 3)
    w0 = torch.tensor([0.2, 0.3, 0.1], dtype=torch.float64, device="cuda", requires_grad=True)
    x0 = Y.clone().requires_grad_(True)
    ptv.tvgen_pdr(x0, w0, [1, 2, 3], [1, 1, 1]).backward(G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        w1 = torch.tensor([0.2, 0.3, 0.1], dtype=torch.float64, device="cuda", requires_grad=True)
        x1 = Y.clone().requires_grad_(True)
        ptv.tvgen_pdr(x1, w1, [1, 2, 3], [1, 1, 1]).backward(G)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(x0.grad, x1.grad) and torch.equal(w0.grad, w1.grad)
    # the C ABI on a non-default stream
    ns, ws, ds = (32, 24, 16), [0.2, 0.3, 0.1], [1, 2, 3]
    yt = flat_buffer(case_input(ns, 4, np.float32), np.float32)
    g = torch.randn_like(yt)
    out0, tape0, _ = record(lib, yt, ns, ws, ds, 3)
    r0 = vjp(lib, tape0, g, ns, ds, 3)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out1, tape1, _ = record(lib, yt, ns, ws, ds, 3, stream=s)
        r1 = vjp(lib, tape1, g, ns, ds, 3, stream=s)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1) and torch.equal(tape0, tape1) and all(torch.equal(p, q) for p, q in zip(r0, r1))
