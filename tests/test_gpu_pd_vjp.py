"""GPU tests (-m gpu) of the PD_TV and PD2_TV backward passes (DESIGN.md section 14): the recorded forward, the unrolled backward and
the torch autograd path of tvgen and tv1_2d(method='pd').

Bars (the device forward's bits and its stop value are never compared with a host driver: the stop value is a grid-dependent
reduction, so info[1] is compared device against device only):
  * recorded forward == proxtv_PD*_TV_dev_* bit for bit, x and info, on the engines seq, chunked, lane and auto, float64 and
    float32, 1D to 4D, 1 to 5 terms and PD2_TV with 1 and 2 terms (a misaligned output forces PD_TV's generic combine), when the
    maxIters cap ends the solve and when the stop rule does (zero penalties: PD_TV at K = 2, PD2_TV at K = 1; a smooth input under
    maxIters = 1000), and the 512 x 512 x 256 float32 volume with 3 terms; the header's K == info[0]; in float64 every recorded
    pass's tape == the host forward's run for the device's K (the oracle's exact prox under seq / chunked, lane_emu.slope_fibers on
    the lane route);
  * backward == the host restatement driven by the device's own tape and K (pd_vjp_emu.backward_from_tapes): gY bit for bit
    (float64 and float32), glam to 1e-12 relative; two identical calls are bit-equal and a NULL glam leaves gY unchanged;
  * refusals write nothing (lambdas included), including a wrong iters and the tapes of the other solvers;
  * autograd: gradcheck and directional differences with the cap binding (K asserted for every evaluation), forward bit-equal to the
    no-grad call, layouts and views, ws as a list / ndarray / tensor and never modified, torch tvgen == numpy tvgen, tv1_2d(method='pd')
    == tvgen with [w, w], a batch axis with the cap binding, a non-default stream.
"""
import ctypes as C

import numpy as np
import pytest

import lane_emu
import pd_vjp_emu as P
from pdr_vjp_emu import exact_prox, slope_prox
from test_gpu_dr2_vjp import kink_free_difference
from test_gpu_pdr_vjp import _a, _p, _st, case_input, flat_buffer, like, volume

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


def name(pd2):
    return "PD2_TV" if pd2 else "PD_TV"


def fn(lib, pd2, what, dt):
    return getattr(lib, "proxtv_%s_%s_dev_%s" % (name(pd2), what, "f32" if dt == torch.float32 else "f64") if what else
                   "proxtv_%s_dev_%s" % (name(pd2), "f32" if dt == torch.float32 else "f64"))


def tape_bytes(lib, pd2, ns, npen, maxit):
    return getattr(lib, "proxtv_%s_tape_bytes" % name(pd2))(_a(np.array(ns, dtype=np.int32)), len(ns), npen, maxit)


def record(lib, pd2, yt, ns, ws, ds, maxit, misaligned=False, stream=None):
    nsa, dsa, lam = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64), np.array(ws, dtype=np.float64)
    nb = tape_bytes(lib, pd2, ns, len(ws), maxit)
    tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    out = like(yt, float("nan"), misaligned)
    info = np.zeros(3)
    f = fn(lib, pd2, "record", yt.dtype)
    assert f(_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _p(tape), nb, _st(stream)) == 1, \
        lib.proxtv_last_error()
    # PD_TV scales lambdas in place like the no-grad call, PD2_TV does not
    assert np.array_equal(lam, np.array(ws, dtype=np.float64) * (1 if pd2 else len(ws)))
    hd = P.header(tape[:256].cpu().numpy())
    assert hd[2] == int(info[0]) and hd[3] == len(ws) and hd[5] == (maxit if maxit > 0 else 35)
    return out, tape, info


def solve(lib, pd2, yt, ns, ws, ds, maxit, misaligned=False):
    nsa, dsa, lam = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64), np.array(ws, dtype=np.float64)
    out = like(yt, float("nan"), misaligned)
    info = np.zeros(3)
    f = fn(lib, pd2, None, yt.dtype)
    assert f(_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(ns), len(ws), maxit, _st()) == 1, lib.proxtv_last_error()
    return out, info


def vjp(lib, pd2, tape, gout, ns, ds, maxit, iters, want_glam=True, stream=None):
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    gY = torch.full_like(gout, float("nan"))
    glam = torch.full((len(ds),), float("nan"), dtype=torch.float64, device="cuda") if want_glam else None
    f = fn(lib, pd2, "vjp", gout.dtype)
    assert f(_a(nsa), len(ns), len(ds), _a(dsa), maxit, iters, _p(tape), _p(gout), _p(gY), _p(glam), _st(stream)) == 1, \
        lib.proxtv_last_error()
    return gY, glam


def check_backward(lib, pd2, tape, G, ns, ds, maxit, K, what):
    """Device backward against the restatement driven by the device's own tape and K."""
    gY, glam = vjp(lib, pd2, tape, torch.tensor(G, device="cuda"), ns, ds, maxit, K)
    hY, hlam = P.backward_from_tapes(P.device_pass_tapes(tape.cpu().numpy(), G.size, len(ds), K, pd2), G, ns, ds, K, pd2)
    assert np.array_equal(gY.cpu().numpy(), hY), what
    g = glam.cpu().numpy()
    assert np.abs(g - hlam).max() <= 1e-12 * max(np.abs(hlam).max(), 1e-300), what


# (pd2, ns, ws, ds): 1D to 4D, 1 to 5 terms, a repeated axis, a zero penalty, an axis without a term; PD2_TV with 1 and 2 terms
CASES = [(False, (3000,), [0.4], [1]),
         (False, (96, 80), [0.3, 0.2], [1, 2]),
         (False, (40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3]),
         (False, (12, 10, 8, 6), [0.3, 0.1, 0.2, 0.4], [1, 2, 3, 4]),
         (False, (20, 18, 16), [0.2, 0.1, 0.3, 0.15, 0.0], [1, 2, 3, 1, 2]),
         (True, (96, 80), [0.3, 0.2], [1, 2]),
         (True, (40, 36, 20), [0.2, 0.25], [3, 1]),
         (True, (3000,), [0.4], [1]),
         (True, (30, 1, 70), [0.3], [3])]


@pytest.mark.parametrize("maxit", [1, 2, 0])
def test_recorded_forward_equals_solve_and_backward(lib, engine, maxit):
    """maxit 1 and 2: the cap ends the solve; 0 (35): the stop rule may end it first.  Either way K = info[0]."""
    for ci, (pd2, ns, ws, ds) in enumerate(CASES):
        for dt in (np.float64, np.float32):
            y = case_input(ns, 3 + ci, dt)
            yt = flat_buffer(y, dt)
            G = np.random.default_rng(ci).normal(size=y.size).astype(dt)
            for eng in ("seq", "chunked", "lane", "auto"):
                engine(eng)
                for mis in ((False, True) if eng == "auto" else (False,)):
                    what = (name(pd2), ns, len(ws), maxit, np.dtype(dt).name, eng, mis)
                    out, tape, info = record(lib, pd2, yt, ns, ws, ds, maxit, misaligned=mis)
                    ref, rinfo = solve(lib, pd2, yt, ns, ws, ds, maxit, misaligned=mis)
                    assert torch.equal(out, ref) and np.array_equal(info, rinfo), what
                    if maxit > 0 and not (pd2 and len(ws) == 1):
                        assert int(info[0]) == maxit, what
                    if eng in ("seq", "auto") and not mis:
                        check_backward(lib, pd2, tape, G, ns, ds, maxit, int(info[0]), what)


def test_stop_rule_ends_the_solve(lib, engine):
    """Zero penalties: PD_TV stops at K = 2 and PD2_TV at K = 1; a smooth input with maxIters = 1000 stops below the cap.  The
    recorded forward equals the solve and the backward follows the device's K."""
    i, j, k = np.meshgrid(np.arange(20), np.arange(18), np.arange(16), indexing="ij")
    smooth3 = (np.sin(i / 5.0) + np.cos(j / 4.0) + np.sin(k / 3.0)).ravel(order="F")
    i2, j2 = np.meshgrid(np.arange(40), np.arange(36), indexing="ij")
    smooth2 = (np.sin(i2 / 7.0) + np.cos(j2 / 5.0)).ravel(order="F")
    cases = [(False, (20, 18, 16), [0.0, 0.0, 0.0], [1, 2, 3], smooth3, 35, 2),
             (True, (40, 36), [0.0, 0.0], [1, 2], smooth2, 35, 1),
             (False, (20, 18, 16), [0.1, 0.1, 0.1], [1, 2, 3], smooth3, 1000, None),
             (False, (40, 36), [0.2, 0.2], [1, 2], smooth2, 1000, None),
             (True, (40, 36), [0.2, 0.2], [1, 2], smooth2, 1000, None)]
    for pd2, ns, ws, ds, y, maxit, Kwant in cases:
        for dt in (np.float64, np.float32):
            yt = flat_buffer(y.astype(dt), dt)
            G = np.random.default_rng(3).normal(size=y.size).astype(dt)
            for eng in ("seq", "auto"):
                engine(eng)
                what = (name(pd2), ns, ws, maxit, np.dtype(dt).name, eng)
                out, tape, info = record(lib, pd2, yt, ns, ws, ds, maxit)
                ref, rinfo = solve(lib, pd2, yt, ns, ws, ds, maxit)
                assert torch.equal(out, ref) and np.array_equal(info, rinfo), what
                K = int(info[0])
                assert (K == Kwant) if Kwant is not None else (1 <= K < maxit), (what, K)
                assert info[1] <= 1e-6, what
                check_backward(lib, pd2, tape, G, ns, ds, maxit, K, what)


@pytest.mark.parametrize("maxit", [2, 0])
def test_tapes_equal_host_forward(lib, engine, port, maxit):
    """float64: under seq / chunked every pass is the exact prox; on the lane route (every axis >= 64 long, >= 1024 fibers) PD_TV's
    passes are the slope-form scan, while PD2_TV's fused inputs (x + p, z + q) keep its passes off the lane route (prox_dispatch.cu
    takes it for plain inputs only), so they stay the exact prox.  The host forward runs the device's K; its output and every pass's
    tape equal the device's."""
    exact = exact_prox(port)
    slope = slope_prox(lane_emu.load())

    def lane_route(a, nf, ln, inc, lam):
        return (slope if lam > 0 and ln >= 64 and nf >= 1024 else exact)(a, nf, ln, inc, lam)
    for pd2, ns, ws, ds, engines in ((False, (40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3], ("seq", "chunked")),
                                     (False, (20, 18, 16), [0.2, 0.1, 0.3, 0.15, 0.0], [1, 2, 3, 1, 2], ("seq", "chunked")),
                                     (True, (96, 80), [0.3, 0.2], [2, 1], ("seq", "chunked")),
                                     (True, (40, 36, 20), [0.3], [2], ("seq", "chunked")),
                                     (False, (64, 64, 64), [0.15, 0.2, 0.25], [1, 2, 3], ("lane",)),
                                     (True, (64, 64, 64), [0.15, 0.2], [1, 3], ("lane",))):
        y = case_input(ns, 7, np.float64)
        yt = flat_buffer(y, np.float64)
        for eng in engines:
            engine(eng)
            out, tape, info = record(lib, pd2, yt, ns, ws, ds, maxit)
            K = int(info[0])
            want, passes = P.forward(lane_route if eng == "lane" and not pd2 else exact, y, ns, ws, ds, K, pd2)
            assert np.array_equal(out.cpu().numpy(), want), (name(pd2), ns, eng)
            host = P.pass_tapes(passes, ns, ws, ds, pd2)
            dev = P.device_pass_tapes(tape.cpu().numpy(), y.size, len(ws), K, pd2)
            assert len(dev) == len(host) == P.n_passes(pd2, len(ws), K)
            for p, ((F, U), (Fh, Uh)) in enumerate(zip(dev, host)):
                assert np.array_equal(F, Fh) and np.array_equal(U, Uh), (name(pd2), ns, eng, p)


def test_volume_512(lib, engine):
    """512 x 512 x 256 float32, 3 terms (BASELINE config 4's volume): the recorded forward equals the solve."""
    import synth_inputs as S
    ns, ws, ds = (512, 512, 256), [0.2, 0.2, 0.2], [1, 2, 3]
    yt = torch.from_numpy(np.ascontiguousarray(S.gen_cfg4(ns, seed=0).ravel(order="F"))).to(device="cuda", dtype=torch.float32)
    engine("auto")
    out, tape, info = record(lib, False, yt, ns, ws, ds, 0)
    ref, rinfo = solve(lib, False, yt, ns, ws, ds, 0)
    assert torch.equal(out, ref) and np.array_equal(info, rinfo)
    assert tape.numel() == 256 + 35 * 3 * 2 * (512 * 512 * 256 // 32 * 4)


def test_backward_deterministic_and_null_glam(lib):
    for pd2, ws, ds in ((False, [0.2, 0.3, 0.25], [1, 2, 3]), (True, [0.2, 0.3], [1, 3])):
        ns = (48, 40, 24)
        y = case_input(ns, 9, np.float64)
        _, tape, info = record(lib, pd2, flat_buffer(y, np.float64), ns, ws, ds, 5)
        K = int(info[0])
        g = torch.randn(y.size, dtype=torch.float64, device="cuda")
        a = vjp(lib, pd2, tape, g, ns, ds, 5, K)
        b = vjp(lib, pd2, tape, g, ns, ds, 5, K)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        assert torch.equal(vjp(lib, pd2, tape, g, ns, ds, 5, K, want_glam=False)[0], a[0])


@pytest.mark.parametrize("pd2", [False, True], ids=["pd", "pd2"])
def test_refusals_write_nothing(lib, pd2):
    ns, K = (20, 16, 12), 3
    ws, ds = ([0.2, 0.3], [1, 3]) if pd2 else ([0.2, 0.3, 0.1], [1, 2, 3])
    npen = len(ws)
    y = case_input(ns, 2, np.float64)
    yt = flat_buffer(y, np.float64)
    _, tape, info = record(lib, pd2, yt, ns, ws, ds, K)
    iters = int(info[0])
    nsa, dsa = np.array(ns, dtype=np.int32), np.array(ds, dtype=np.float64)
    nb = tape_bytes(lib, pd2, ns, npen, K)
    assert nb == 256 + (2 * K if pd2 else K * npen) * 2 * (((y.size + 31) // 32 * 4 + 255) // 256 * 256)
    assert tape_bytes(lib, True, ns, 1, K) == 256 + 2 * (((y.size + 31) // 32 * 4 + 255) // 256 * 256)
    assert tape_bytes(lib, True, ns, 3, K) == 0 and tape_bytes(lib, False, ns, 65, K) == 0
    # a capacity whose pass count passes 2^32 (3 x 1431655766 = 2^32 + 2): the size is exact, and a buffer of the wrapped size is short
    huge = 1431655766
    sb2 = 2 * (((y.size + 31) // 32 * 4 + 255) // 256 * 256)
    assert tape_bytes(lib, pd2, ns, npen, huge) == 256 + (2 * huge if pd2 else huge * npen) * sb2
    wrapped = 256 + 2 * sb2
    rec = fn(lib, pd2, "record", torch.float64)
    o = torch.full_like(yt, 3.0)
    t2 = torch.full((nb,), 7, dtype=torch.uint8, device="cuda")
    info = np.zeros(3)
    lam0 = np.array(ws)
    big = np.arange(1, 66, dtype=np.float64) % 3 + 1
    lam65 = np.full(65, 0.1)
    neg = lam0.copy(); neg[1] = -0.3
    bad = [dict(y=None), dict(x=None), dict(lam=None), dict(dims=None), dict(ns=None), dict(tape=None),
           dict(nds=0), dict(nds=17), dict(ns=np.array([20, -16, 12], dtype=np.int32)), dict(npen=0),
           dict(npen=65, lam=lam65, dims=big), dict(dims=np.array([1.0, 4.0, 2.0])), dict(dims=np.array([0.0, 2.0, 3.0])),
           dict(lam=neg), dict(tb=nb - 1), dict(maxit=huge, tb=wrapped),
           dict(ns=np.array([1 << 15] * 3, dtype=np.int32), maxit=2 ** 31 - 1)]          # a tape size past 2^64 bytes
    if pd2:
        bad.append(dict(npen=3, lam=np.array([0.2, 0.3, 0.1]), dims=np.array([1.0, 2.0, 3.0])))
    for i, kw in enumerate(bad):
        lam = kw.get("lam", lam0).copy() if kw.get("lam", lam0) is not None else None
        nsx = kw.get("ns", nsa)
        nds = kw.get("nds", 3)
        nsx17 = np.full(17, 1, dtype=np.int32) if nds == 17 else nsx
        info[:] = 0
        r = rec(_p(kw.get("y", yt)), _a(lam), _a(kw.get("dims", dsa)), _p(kw.get("x", o)), _a(info), _a(nsx17), nds,
                kw.get("npen", npen), kw.get("maxit", K), _p(kw.get("tape", t2)), kw.get("tb", nb), None)
        assert r == 0 and info[2] == 3, i
        if lam is not None:
            assert np.array_equal(lam, kw.get("lam", lam0)), i                  # not scaled
    # vjp refusals: NULL arrays, another iteration count, capacity, dtype, shape, axes or term count, the other solvers' tapes
    g = torch.randn_like(yt)
    gY = torch.full_like(g, 3.0)
    glam = torch.full((npen,), 3.0, dtype=torch.float64, device="cuda")
    vf = fn(lib, pd2, "vjp", torch.float64)

    def call(f=vf, nsx=nsa, nds=3, npen=npen, dims=dsa, k=K, it=iters, tp=tape, gg=g, gy=gY):
        return f(_a(nsx), nds, npen, _a(dims), k, it, _p(tp), _p(gg), _p(gy), _p(glam), None)
    assert call(it=iters + 1) == 0 and call(it=iters - 1) == 0 and call(it=-1) == 0
    assert call(k=K + 1) == 0 and call(k=0) == 0
    assert call(nsx=np.array([20, 12, 16], dtype=np.int32)) == 0
    assert call(dims=dsa[::-1].copy()) == 0
    assert call(npen=npen - 1) == 0 and call(nds=2) == 0
    assert call(tp=None) == 0 and call(gg=None) == 0 and call(gy=None) == 0
    g32 = g.float(); gY32 = torch.full_like(g32, 3.0)
    assert call(f=fn(lib, pd2, "vjp", torch.float32), gg=g32, gy=gY32) == 0                # recorded in float64
    # the tapes of PDR_TV, of the other Dykstra solver, of DR2_TV and of DR2L1W_TV (same shape where they have one)
    others = []
    lamx = np.array(ws, dtype=np.float64)
    o2 = torch.empty_like(yt)
    pdr = torch.zeros(lib.proxtv_PDR_TV_tape_bytes(_a(nsa), 3, npen, K), dtype=torch.uint8, device="cuda")
    assert lib.proxtv_PDR_TV_record_dev_f64(_p(yt), _a(lamx.copy()), _a(dsa), _p(o2), None, _a(nsa), 3, npen, K, _p(pdr), pdr.numel(),
                                            None) == 1
    others.append(pdr)
    _, t_other, _ = record(lib, not pd2, yt, ns, ws[:2], ds[:2], K)        # the other Dykstra solver, 2 terms
    others.append(t_other)
    M, N = 20, 192                                                                      # the same number of elements as an image
    dr2 = torch.zeros(lib.proxtv_DR2_TV_tape_bytes(M, N, 1, K), dtype=torch.uint8, device="cuda")
    assert lib.proxtv_DR2_TV_record_dev_f64(M, N, 1, 0, _p(yt), 0.3, 0.3, _p(o2), K, _p(dr2), dr2.numel(), None, None) == 1
    drw = torch.zeros(lib.proxtv_DR2L1W_TV_tape_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    w1 = torch.full(((M - 1) * N,), 0.2, dtype=torch.float64, device="cuda")
    w2 = torch.full((M * (N - 1),), 0.2, dtype=torch.float64, device="cuda")
    assert lib.proxtv_DR2L1W_TV_record_dev_f64(M, N, _p(yt), _p(w1), _p(w2), _p(o2), K, _p(drw), drw.numel(), None, None) == 1
    others += [dr2, drw]
    for other in others:
        big_enough = torch.zeros(max(other.numel(), nb), dtype=torch.uint8, device="cuda")
        big_enough[:other.numel()] = other
        assert call(tp=big_enough) == 0
    torch.cuda.synchronize()
    assert bool((o == 3.0).all()) and bool((t2 == 7).all())
    assert bool((gY == 3.0).all()) and bool((glam == 3.0).all()) and bool((gY32 == 3.0).all())


# ---------------------------------------------------------------------------------------------------------------- autograd
def capped(ptv, f, K):
    """f, asserting after every evaluation that the cap ended the solve (K == max_iters): no step of a difference changes K."""
    def g(*a):
        out = f(*a)
        assert ptv.tvgen.last_info[0] == K
        return out
    return g


def test_gradcheck(ptv, engine):
    for eng in ("auto", "seq"):
        engine(eng)
        x = volume((6, 5, 4), 21).requires_grad_(True)
        w = torch.tensor([0.2, 0.3, 0.25], dtype=torch.float64, device="cuda", requires_grad=True)
        f = capped(ptv, lambda a, b: ptv.tvgen(a, b, [1, 2, 3], [1, 1, 1], max_iters=3), 3)
        assert torch.autograd.gradcheck(f, (x, w), eps=1e-6, atol=1e-6)
        x2 = volume((9, 7), 22).requires_grad_(True)
        w2 = torch.tensor([0.3, 0.2], dtype=torch.float64, device="cuda", requires_grad=True)
        f2 = capped(ptv, lambda a, b: ptv.tvgen(a, b, [1, 2], [1, 1], max_iters=3), 3)
        assert torch.autograd.gradcheck(f2, (x2, w2), eps=1e-6, atol=1e-6)
        x3 = volume((7, 6), 23).requires_grad_(True)
        w3 = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
        f3 = capped(ptv, lambda a, b: ptv.tv1_2d(a, b, max_iters=2, method="pd"), 2)
        assert torch.autograd.gradcheck(f3, (x3, w3), eps=1e-6, atol=1e-6)


def test_directional_differences(ptv):
    """A few iterations on noise with the cap binding (asserted for every evaluation)."""
    for shape, ws, ds, K in (((40, 36, 20), [0.2, 0.25, 0.3], [1, 2, 3], 4), ((96, 64), [0.3, 0.2], [1, 2], 4)):
        Y = volume(shape, 8)
        G = volume(shape, 9)
        x = Y.clone().requires_grad_(True)
        w = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
        fn_ = capped(ptv, lambda a, b, ds=ds, K=K: ptv.tvgen(a, b, ds, [1] * len(ds), max_iters=K), K)
        (fn_(x, w) * G).sum().backward()
        with torch.no_grad():
            base = fn_(Y, ws)
            V = volume(shape, 10)
            fd = kink_free_difference(lambda e: ((fn_(Y + e * V, ws) - base) * G).sum().item())
            an = (x.grad * V).sum().item()
            assert abs(fd - an) <= 2e-6 * max(abs(an), 1.0), (shape, fd, an)
            for i in range(len(ws)):
                def step(e):
                    wh = list(ws); wh[i] += e
                    return ((fn_(Y, wh) - base) * G).sum().item()
                fdw = kink_free_difference(step)
                assert abs(fdw - w.grad[i].item()) <= 2e-6 * max(abs(fdw), 1.0), (shape, i, fdw, w.grad[i].item())


@pytest.mark.parametrize("ws", [[0.25, 0.375, 0.125], [0.25, 0.375]], ids=["pd", "pd2"])
def test_forward_equals_no_grad_layouts_and_ws(ptv, engine, ws):
    """C order, Fortran order and a non-contiguous view; ws as a list, an ndarray and tensors of two dtypes and devices (never
    modified); the result keeps x's memory order.  The penalties are exact in float32, so every form of ws carries the same values."""
    ds = [1, 2, 3][:len(ws)]
    for eng in ("seq", "auto"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            Y = volume((24, 20, 16), 4, dt)
            G = volume((24, 20, 16), 5, dt)
            ref = ptv.tvgen(Y, ws, ds, [1] * len(ws))
            K = ptv.tvgen.last_info[0]
            assert ref.grad_fn is None and ref.is_contiguous()
            grads = []
            for make in (lambda: Y.clone(), lambda: Y.permute(2, 1, 0).contiguous().permute(2, 1, 0),
                         lambda: torch.nn.functional.pad(Y, (0, 3))[:, :, :16]):
                v = make()
                no_grad = ptv.tvgen(v, ws, ds, [1] * len(ws))
                info0 = ptv.tvgen.last_info.copy()
                x = v.detach().requires_grad_(True)
                out = ptv.tvgen(x, ws, ds, [1] * len(ws))
                assert out.grad_fn is not None and torch.equal(out.detach(), no_grad), (eng, dt)
                assert np.array_equal(ptv.tvgen.last_info, info0)
                if eng == "seq":
                    assert torch.equal(no_grad, ref) and info0[0] == K, (eng, dt, v.stride())
                assert out.stride() == (v.stride() if (v.is_contiguous() or ptv._f_contiguous(v)) else ref.stride())
                out.backward(G)
                grads.append(x.grad)
            if eng == "seq":
                assert all(torch.equal(g, grads[0]) for g in grads)
            with torch.no_grad():
                assert ptv.tvgen(Y.clone().requires_grad_(True), ws, ds, [1] * len(ws)).grad_fn is None
            wl, wa = list(ws), np.array(ws)
            wt64 = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
            wt32 = torch.tensor(ws, dtype=torch.float32, requires_grad=True)                  # float32 on the CPU
            res = []
            for w in (wl, wa, wt64, wt32):
                x = Y.clone().requires_grad_(True)
                out = ptv.tvgen(x, w, ds, [1] * len(ws))
                out.backward(G)
                res.append((out.detach(), x.grad))
            assert all(torch.equal(r[0], res[0][0]) and torch.equal(r[1], res[0][1]) for r in res)
            assert wl == ws and np.array_equal(wa, ws) and torch.equal(wt64.detach().cpu(), torch.tensor(ws, dtype=torch.float64))
            assert wt32.grad.dtype == torch.float32 and wt32.grad.device.type == "cpu"
            assert torch.equal(wt32.grad, wt64.grad.cpu().float())


@pytest.mark.parametrize("ws,ds", [([0.3, 0.2, 0.25], [1, 2, 3]), ([0.3, 0.2], [1, 3]), ([0.3, 0.2, 0.1, 0.2], [1, 2, 3, 1])],
                         ids=["pd", "pd2", "pd-4terms"])
def test_torch_equals_numpy(ptv, engine, ws, ds):
    """float64, the same K (the cap ends every solve, asserted): an F-ordered tensor takes the numpy path's routes, bit for bit on
    every engine; a C-ordered tensor has other fiber strides, bit for bit under seq / chunked, to 1e-12 under auto."""
    rng = np.random.default_rng(12)
    A = rng.normal(size=(30, 24, 20))
    K = 6
    for eng in ("seq", "chunked", "lane", "auto"):
        engine(eng)
        want = ptv.tvgen(np.asfortranarray(A), list(ws), ds, [1] * len(ws), max_iters=K)
        assert ptv.tvgen.last_info[0] == K, eng
        tF = torch.tensor(np.asfortranarray(A), device="cuda").permute(2, 1, 0).contiguous().permute(2, 1, 0)
        assert ptv._f_contiguous(tF) and not tF.is_contiguous()
        gotF = ptv.tvgen(tF, list(ws), ds, [1] * len(ws), max_iters=K)
        assert ptv.tvgen.last_info[0] == K and np.array_equal(gotF.cpu().numpy(), want), eng
        gotC = ptv.tvgen(torch.tensor(A, device="cuda"), list(ws), ds, [1] * len(ws), max_iters=K)
        assert ptv.tvgen.last_info[0] == K, eng
        if eng in ("seq", "chunked"):
            assert np.array_equal(gotC.cpu().numpy(), want), eng
        else:
            assert np.abs(gotC.cpu().numpy() - want).max() <= 1e-12 * np.abs(want).max(), eng


def test_tv1_2d_pd_equals_tvgen(ptv):
    for dt in (torch.float64, torch.float32):
        Y = volume((70, 50), 13, dt)
        G = volume((70, 50), 14, dt)
        res = []
        for via in ("tv1_2d", "tvgen"):
            x = Y.clone().requires_grad_(True)
            w = torch.tensor(0.3, dtype=torch.float64, device="cuda", requires_grad=True)
            if via == "tv1_2d":
                out = ptv.tv1_2d(x, w, method="pd")
            else:
                out = ptv.tvgen(x, torch.stack([w, w]), [1, 2], [1, 1])
            out.backward(G)
            res.append((out.detach(), x.grad, w.grad))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
        assert abs(res[0][2].item() - res[1][2].item()) <= 1e-12 * abs(res[1][2].item())
        assert torch.equal(ptv.tv1_2d(Y, 0.3, method="pd"), res[0][0])
        assert torch.equal(ptv.tv1_2d(Y, 0.3, method="pd"), ptv.tvgen(Y, [0.3, 0.3], [1, 2], [1, 1]))
    with pytest.raises(AssertionError):                # one penalty for both terms: a number or a 0-dim tensor
        ptv.tv1_2d(Y, torch.tensor([0.3], dtype=torch.float64, device="cuda", requires_grad=True), method="pd")


def test_batch_axis_equals_slices_when_capped(ptv, engine):
    """A leading batch axis without a term equals the per-slice solves and gradients bit for bit only when the cap ends every solve
    (the stop test is global); K == max_iters is asserted."""
    for eng in ("seq", "chunked"):
        engine(eng)
        for dt in (torch.float64, torch.float32):
            for ws, ds in (([0.3, 0.2, 0.1], [2, 3, 3]), ([0.3, 0.2], [2, 3])):
                X = volume((3, 40, 72), 6, dt)
                G = volume((3, 40, 72), 7, dt)
                x = X.clone().requires_grad_(True)
                out = ptv.tvgen(x, ws, ds, [1] * len(ws), max_iters=4)
                assert ptv.tvgen.last_info[0] == 4
                out.backward(G)
                for b in range(3):
                    xb = X[b].clone().requires_grad_(True)
                    ob = ptv.tvgen(xb, ws, [d - 1 for d in ds], [1] * len(ws), max_iters=4)
                    assert ptv.tvgen.last_info[0] == 4
                    ob.backward(G[b])
                    assert torch.equal(ob.detach(), out.detach()[b]) and torch.equal(xb.grad, x.grad[b]), (eng, dt, b)


def test_non_default_stream(ptv, lib):
    Y, G = volume((32, 24, 16), 2), volume((32, 24, 16), 3)
    for ws in ([0.2, 0.3, 0.1], [0.2, 0.3]):
        ds = [1, 2, 3][:len(ws)]
        w0 = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
        x0 = Y.clone().requires_grad_(True)
        ptv.tvgen(x0, w0, ds, [1] * len(ws)).backward(G)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            w1 = torch.tensor(ws, dtype=torch.float64, device="cuda", requires_grad=True)
            x1 = Y.clone().requires_grad_(True)
            ptv.tvgen(x1, w1, ds, [1] * len(ws)).backward(G)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        assert torch.equal(x0.grad, x1.grad) and torch.equal(w0.grad, w1.grad)
    # the C ABI on a non-default stream
    ns, ws, ds = (32, 24, 16), [0.2, 0.3, 0.1], [1, 2, 3]
    yt = flat_buffer(case_input(ns, 4, np.float32), np.float32)
    g = torch.randn_like(yt)
    out0, tape0, info0 = record(lib, False, yt, ns, ws, ds, 3)
    r0 = vjp(lib, False, tape0, g, ns, ds, 3, int(info0[0]))
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out1, tape1, info1 = record(lib, False, yt, ns, ws, ds, 3, stream=s)
        r1 = vjp(lib, False, tape1, g, ns, ds, 3, int(info1[0]), stream=s)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1) and torch.equal(tape0, tape1) and all(torch.equal(p, q) for p, q in zip(r0, r1))
