"""GPU tests (-m gpu) of the single-item N-D TV-L1 prox -- PDR_TV (proxtv_PDR_TV_dev_*, tvgen_pdr) and PD_TV / PD2_TV, which run as a
batch of one (proxtv_PD_TV_dev_* / proxtv_PD2_TV_dev_*, tvgen) -- against the float64 oracle (orc_pdr_tv / orc_pd_tv / orc_pd2_tv) on
every fiber route their prox passes take.

The route of a term is test_gpu_nd_routes.Case.term_route at m = 1: one item of shape ns, column-major, whose term i runs one call of
prox_fibers_ex on (nf, ns[d], prod(ns[:d])) with 3 n elements of scratch.  PDR_TV is that restatement with the flag of PD_TV (pd2
False): it scales the penalties by npen, reads a plain input (z_i), so its passes may take the lane engine, and never uses the fused
x + p input.  A single item has no batch to lose items from, so a term keeps its route for the whole solve, and the lane engine is
reached only when the item alone has >= 1024 fibers of >= 64 samples.  Each case id names the route of every term.  What the library
shows of the routes -- the contiguous- and strided-scan launch counters, proxtv_lane_guard_last, proxtv_long_fiber_last -- is checked
by test_gpu_nd_routes.check_routes.

Bars:
  * PDR_TV, float64, every route (lane included), at the default count (0: 35 iterations), 20 and 40: relerr(x, orc_pdr_tv) <= 1e-9;
    info[0] == the count; info[1] within 1e-9 relative of the oracle's stop value; info[2] == RC_ITERS exactly when the count is >= 35.
    The lane route, 35 lane passes per term, measured at most 1.8e-13 relative to the oracle on an H100 (80 GB, default power limit);
  * PDR_TV, float32, 35 iterations: relerr against the float64 oracle on the float32-rounded input <= F32_PDR_BAR = 5.5e-4.  The bar
    comes from the seq engine, where every pass is the exact taut-string scan in float32: its largest error over these cases was
    1.1e-4 (p1hi; p1, the same data at a tenth of the penalty, 5.8e-5; the other cases 5e-7 .. 9e-6) on an H100 (80 GB, default power
    limit), and the bar gives it a margin of 5x; the seq engine is held to a quarter of the bar so that the margin cannot erode
    unnoticed.  The other routes measured no more than the seq engine on the same case (the lane engine, which scans in double and
    rounds once, 5.6e-5 on p1).  The float32 error of PDR_TV is much larger than PD_TV's at 8 iterations (test_gpu_nd_routes.F32_BAR):
    it runs 35 iterations, and it grows with the penalty;
  * PD_TV / PD2_TV: float64 relerr <= 1e-9 and K == the oracle's wherever test_gpu_nd_routes.check_K's margin decides it; float32 at
    maxIters = 8 within test_gpu_nd_routes.F32_BAR, the batched solvers' bar;
  * the exact engines (seq, chunked, chunked-strided) give x and info bit for bit equal to seq's, in both dtypes: every non-lane route
    is the sequential Scan<T>, and the combine does not depend on the engine;
  * an output one element into a larger buffer (not 16-byte aligned; float32: not 8-byte aligned) changes the combine (PD_TV and
    PDR_TV: the generic kernel) or, PD2_TV in float32, the strided passes' gather / scatter tiles: x is bit for bit the aligned call's
    and K equal; the stop value differs only by reduction order (<= 1e-12 relative; PD2_TV: bit-equal), and a NULL info leaves x as it was;
  * the device entry on a side stream, the host entries (PDR_TV, PD_TV, PD2_TV, proxtv_PD_TV_f32), tvgen / tvgen_pdr on numpy and on
    C- and Fortran-ordered tensors and tv1_2d(method='pd') are bit for bit the device entry under the chunked engine.  The C ABI (host
    and device) scales PD_TV's and PDR_TV's penalties in place, as the reference does, so every call gets a fresh array; the torch
    paths never write ws.
"""
import ctypes as C
import time

import numpy as np
import pytest

from conftest import relerr
from test_gpu_nd_routes import (ENGINES, EXACT_ENGINES, F32_BAR, F32_MAXIT, Case, check_K, check_routes, counters,
                                reset_long_fiber_hook)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32_PDR_BAR = 5.5e-4                # float32 PDR_TV relerr against the oracle: 5x the largest seen on the seq route (module docstring)
PDR_COUNTS = (0, 20, 40)            # the default (35), one cap below it and one above
RC_OK, RC_ITERS = 0, 1              # ptv_internal.h
DEFAULT_ITERS = 35                  # MAX_ITERS_DR / MAX_ITERS_PD


class Single(Case):
    """One item of one solver: "PDR" (pd2 False: penalties times npen, plain input), "PD" or "PD2"."""

    def __init__(self, key, solver, ns, ds, ws, kind, maxit, engines=ENGINES):
        super().__init__(key, solver == "PD2", ns, ds, ws, [kind], maxit, engines)
        self.solver = solver

    def id(self, engine, dt):
        routes = "+".join("%d:%s" % (self.ds[i], self.term_route(i, 1, dt, engine)) for i in range(len(self.ws)))
        return "%s-%s-%s-%s-%s-%s" % (self.key, self.solver, np.dtype(dt).name, "x".join(map(str, self.ns)), engine, routes)


CASES = [
    # 1536 fibers on axes 1 and 2: the lane engine (contiguous and strided) on one item; axis 3 is shorter than 64: sequential
    Single("p1", "PDR", (64, 64, 24), [1, 2, 3], [0.1, 0.1, 0.1], "noisy", 0),
    # chunked (axis 1, 80 fibers) and the sparse gather / scatter (axis 2, inc 96); the direct strided kernel under chunked-strided
    Single("p2", "PDR", (96, 80), [1, 2], [0.2, 0.25], "noisy", 0),
    # row pitch 129 * 8 = 1032 bytes (129 * 4 = 516), not a multiple of 16: the lane engine refuses axes 1 and 2 though both have
    # >= 1024 fibers; inc 129 is odd: no direct strided kernel, the gather / scatter under every engine but seq; axis 1 repeated
    Single("p3", "PDR", (129, 70, 16), [1, 2, 1], [0.1, 0.15, 0.1], "noisy", 0),
    # strided fibers longer than the chunked kernel takes: gathered, then the sequential kernel
    Single("p4", "PDR", (2, 33000), [2], [0.3], "noisy", 0),
    # one contiguous fiber longer than the chunked kernel takes: the long-fiber tiles (3 n >= lf_scratch_elems); on this input their
    # agreement check fails and the pass falls back to the sequential kernel (long-fallback)
    Single("p5", "PDR", (40000,), [1], [0.3], "smooth~0.05", 0),
    # five terms: the generic combine; axes 1 and 2 repeated
    Single("p6", "PDR", (70, 66, 9), [1, 2, 3, 2, 1], [0.1, 0.2, 0.15, 0.05, 0.1], "noisy", 0),
    # n = 7777, odd: the vector combine's scalar tail (1 element in float64, 1 in float32)
    Single("p7", "PDR", (101, 77), [2, 1], [0.3, 0.2], "smooth~0.05", 0),
    # the guard's other decision: penalties above the mean step of p1's input (the lane route otherwise)
    # (and, under seq, the largest float32 error of the table: the bar's measurement)
    Single("p1hi", "PDR", (64, 64, 24), [1, 2, 3], [1.0, 1.0, 1.0], "noisy", 0, engines=("seq", "auto")),
    # PD_TV on one item with >= 1024 fibers per axis: the lane engine at m = 1, contiguous and strided, and the guard both ways
    Single("s1", "PD", (64, 64, 24), [1, 2, 3], [0.1, 0.1, 0.1], "noisy", 40),
    Single("s1hi", "PD", (64, 64, 24), [1, 2, 3], [1.0, 1.0, 1.0], "noisy", 40, engines=("auto",)),
    # PD2_TV: the fused x + p input through the chunked contiguous kernel and the sparse gather / scatter
    Single("s2", "PD2", (96, 80), [1, 2], [0.2, 0.25], "noisy", 20),
    # PD2_TV with a smooth item that stops on its own: K decided by the stop test
    Single("s3", "PD2", (96, 80), [1, 2], [0.2, 0.25], "smooth~0.02", 60),
]
CASE_BY_KEY = {c.key: c for c in CASES}
PARAMS = [(c, e) for c in CASES for e in c.engines]
IDS64 = [c.id(e, np.float64) for c, e in PARAMS]
IDS32 = [c.id(e, np.float32) for c, e in PARAMS]
SEEN = {"routes": set(), "guard": set(), "ran64": 0, "ran32": 0, "t0": None, "f32_err": {}, "f32_seq": {}, "f32_case": {}, "lane_err": 0.0}


# ---- the oracle, once per case, dtype and count -----------------------------------------------------------------------------
_ORACLE = {}


def oracle(port, case, dt, maxit):
    """[(x in float64, flat; K; stop after K; stop after K - 1, or inf when K == 1 or for PDR_TV)] for the one item, as
    test_gpu_nd_routes.check_K takes it; float32: the float64 oracle on the float32-rounded input."""
    key = (case.key, np.dtype(dt).name, maxit)
    if key not in _ORACLE:
        fn = {"PDR": port.pdr_tv, "PD": port.pd_tv, "PD2": port.pd2_tv}[case.solver]
        V = case.Y(dt).astype(np.float64).reshape(case.ns, order="F")
        x, info = fn(V, list(case.ws), case.ds, maxit=maxit)
        K = int(info[0])
        prev = fn(V, list(case.ws), case.ds, maxit=K - 1)[1][1] if K > 1 and case.solver != "PDR" else np.inf
        _ORACLE[key] = ([(x.ravel(order="F"), K, float(info[1]), float(prev))], info)
    return _ORACLE[key]


# ---- calls ----------------------------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr())


def _a(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def sfx(dt):
    return "f32" if dt in (np.float32, torch.float32) else "f64"


def scaled(case):
    """The penalties as the C ABI leaves them: times npen for PD_TV and PDR_TV (in place, like the reference), as given for PD2_TV."""
    return np.array(case.ws, dtype=np.float64) * (1 if case.pd2 else len(case.ws))


def dev(lib, case, yt, maxit, misaligned=False, with_info=True, stream=None):
    """proxtv_<solver>_dev_* on the flat tensor yt into a fresh NaN buffer (misaligned: one element into a larger one); (out, info)."""
    lam, dsa, nsa = np.array(case.ws, dtype=np.float64), np.array(case.ds, dtype=np.float64), np.array(case.ns, dtype=np.int32)
    buf = torch.full((case.n + (1 if misaligned else 0),), float("nan"), dtype=yt.dtype, device="cuda")
    out = buf[1:] if misaligned else buf
    info = np.zeros(3) if with_info else None
    f = getattr(lib, "proxtv_%s_TV_dev_%s" % (case.solver, sfx(yt.dtype)))
    args = [_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(case.ns), len(case.ws), maxit]
    if stream is None:
        assert f(*args, C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 1, lib.proxtv_last_error()
    else:
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            assert f(*args, C.c_void_p(stream.cuda_stream)) == 1, lib.proxtv_last_error()
        stream.synchronize()
    assert np.array_equal(lam, scaled(case)), ("the penalties as the call left them", lam, case.ws)
    return out, info


@pytest.fixture
def lib(ptv):
    L = ptv.load()
    prev = ptv.set_engine("auto")
    yield L
    ptv.set_engine(prev)
    L.proxtv_profile_reset()


# ---- checks -------------------------------------------------------------------------------------------------------------------
def count_of(maxit):
    return maxit if maxit > 0 else DEFAULT_ITERS


def check_info(case, info, orc, oinfo, dt, maxit):
    """PDR_TV: the count, its stop value and return code; PD_TV / PD2_TV: K against the oracle's (check_K)."""
    if case.solver == "PDR":
        n = count_of(maxit)
        assert info[0] == n and oinfo[0] == n, (info, oinfo)
        assert info[2] == (RC_ITERS if n >= DEFAULT_ITERS else RC_OK) == oinfo[2], (info, oinfo)
        if dt == np.float64:
            assert abs(info[1] - oinfo[1]) <= 1e-9 * abs(oinfo[1]), ("stop value", info[1], oinfo[1])
    else:
        check_K(case, info.reshape(1, 3), orc, dt, maxit)
        assert info[2] == (RC_ITERS if info[0] >= DEFAULT_ITERS else RC_OK), info


def f32_bar(case):
    return F32_PDR_BAR if case.solver == "PDR" else F32_BAR


def f32_maxit(case):
    return 0 if case.solver == "PDR" else F32_MAXIT


def f64_counts(case):
    return PDR_COUNTS if case.solver == "PDR" else (case.maxit,)


def run_case(ptv, port, lib, case, engine, dt, maxit):
    """One solve under the engine with its routes checked; (input tensor, out, info, error against the oracle, route names)."""
    guard, gmargin = case.guard(dt)
    if engine == "auto":
        assert gmargin > 1e-6, "the data sits on the lane guard's threshold"
    orc, oinfo = oracle(port, case, dt, maxit)
    Yt = torch.tensor(case.Y(dt), device="cuda")
    ptv.set_engine(engine)
    reset_long_fiber_hook(lib)
    lib.proxtv_profile_reset()
    out, info = dev(lib, case, Yt, maxit)
    launches = counters(lib)
    if engine == "auto":
        assert lib.proxtv_lane_guard_last() == int(guard), (lib.proxtv_lane_guard_last(), guard)
        SEEN["guard"].add(int(guard))
    check_info(case, info, orc, oinfo, dt, maxit)
    names = check_routes(lib, case, dt, engine, info.reshape(1, 3), launches, guard)
    err = relerr(out.double().cpu().numpy(), orc[0][0])
    return Yt, out, info, err, names


def check_exact(ptv, lib, case, engine, Yt, out, info, maxit):
    """chunked and chunked-strided: x and info bit for bit the seq engine's."""
    if engine in EXACT_ENGINES and engine != "seq":
        ptv.set_engine("seq")
        sout, sinfo = dev(lib, case, Yt, maxit)
        assert torch.equal(out, sout) and np.array_equal(info, sinfo), ("not the seq engine's result", info, sinfo)


@pytest.mark.parametrize("case,engine", PARAMS, ids=IDS64)
def test_forward_f64(ptv, port, lib, case, engine):
    if SEEN["t0"] is None:
        SEEN["t0"] = time.perf_counter()
    for maxit in f64_counts(case):
        Yt, out, info, err, names = run_case(ptv, port, lib, case, engine, np.float64, maxit)
        assert err <= 1e-9, (maxit, err)
        if "lane" in names:
            SEEN["lane_err"] = max(SEEN["lane_err"], err)
        check_exact(ptv, lib, case, engine, Yt, out, info, maxit)
        SEEN["routes"] |= names
    SEEN["ran64"] += 1


@pytest.mark.parametrize("case,engine", PARAMS, ids=IDS32)
def test_forward_f32(ptv, port, lib, case, engine):
    maxit = f32_maxit(case)
    Yt, out, info, err, names = run_case(ptv, port, lib, case, engine, np.float32, maxit)
    bar = f32_bar(case)
    SEEN["f32_case"][case.key] = max(SEEN["f32_case"].get(case.key, 0.0), err)
    for r in names:
        SEEN["f32_err"][(case.solver, r)] = max(SEEN["f32_err"].get((case.solver, r), 0.0), err)
    assert err <= bar, (err, bar)
    if engine == "seq":
        SEEN["f32_seq"][case.solver] = max(SEEN["f32_seq"].get(case.solver, 0.0), err)
        assert err <= bar / 4, ("the float32 bar no longer has its margin over the seq route", err)
    check_exact(ptv, lib, case, engine, Yt, out, info, maxit)
    SEEN["routes"] |= names
    SEEN["ran32"] += 1


# ---- the output's alignment -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["float64", "float32"])
@pytest.mark.parametrize("key", ["p2", "p6", "p7", "s1", "s2"])
def test_misaligned_output(ptv, port, lib, key, dt):
    """x one element into a larger buffer: the same x bit for bit, the same K, the stop value up to its reduction order, within the
    oracle's bar; a NULL info leaves x as it was.  The strided terms take the gather / scatter under the chunked engine."""
    case = CASE_BY_KEY[key]
    maxit = case.maxit if dt == np.float64 else f32_maxit(case)
    ptv.set_engine("chunked")
    Yt = torch.tensor(case.Y(dt), device="cuda")
    out, info = dev(lib, case, Yt, maxit)
    mout, minfo = dev(lib, case, Yt, maxit, misaligned=True)
    assert mout.data_ptr() % 8 != 0 if dt == np.float32 else mout.data_ptr() % 16 != 0
    assert torch.equal(mout, out), "the misaligned output changed x"
    assert minfo[0] == info[0] and minfo[2] == info[2], (minfo, info)
    if case.pd2:
        assert minfo[1] == info[1], (minfo, info)
    else:
        assert abs(minfo[1] - info[1]) <= 1e-12 * abs(info[1]), (minfo, info)
    orc, oinfo = oracle(port, case, dt, maxit)
    check_info(case, minfo, orc, oinfo, dt, maxit)
    assert relerr(mout.double().cpu().numpy(), orc[0][0]) <= (1e-9 if dt == np.float64 else f32_bar(case))
    for mis in (False, True):
        nout, _ = dev(lib, case, Yt, maxit, misaligned=mis, with_info=False)
        assert torch.equal(nout, out), ("NULL info", mis)


# ---- the other entry points ---------------------------------------------------------------------------------------------------
def flat_of(t):
    """The column-major flat array of a result of shape ns, whatever its strides."""
    return t.permute(tuple(range(t.dim() - 1, -1, -1))).reshape(-1)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["float64", "float32"])
@pytest.mark.parametrize("key", ["p2", "p6", "s1", "s2"])
def test_entries(ptv, port, lib, key, dt):
    """Under the chunked engine, bit for bit the device entry: the device entry on a side stream, the host entry, tvgen / tvgen_pdr on
    numpy and on C- and Fortran-ordered tensors; the penalties scaled in place by the C ABI and never written by the torch paths."""
    case = CASE_BY_KEY[key]
    maxit = case.maxit if dt == np.float64 else f32_maxit(case)
    nd, k = len(case.ns), len(case.ws)
    ptv.set_engine("chunked")
    Y = case.Y(dt)
    Yt = torch.tensor(Y, device="cuda")
    out, info = dev(lib, case, Yt, maxit)
    want = out.cpu().numpy()
    sout, sinfo = dev(lib, case, Yt, maxit, stream=torch.cuda.Stream())
    assert torch.equal(sout, out) and np.array_equal(sinfo, info), "side stream"
    front = ptv.tvgen_pdr if case.solver == "PDR" else ptv.tvgen
    if dt == np.float64 or case.solver == "PD":                  # float32 has a host entry for PD_TV only, proxtv_PD_TV_f32
        # the host entries: the reference's symbols in float64
        lam, dsa, nsa = np.array(case.ws, dtype=np.float64), np.array(case.ds, dtype=np.float64), np.array(case.ns, dtype=np.int32)
        hout, hinfo = np.full_like(Y, np.nan), np.zeros(3)
        if dt == np.float64:
            rc = getattr(lib, "%s_TV" % case.solver)(_a(Y), _a(lam), _a(np.ones(k)), _a(dsa), _a(hout), _a(hinfo), _a(nsa), nd, k, 1, maxit)
        else:
            rc = lib.proxtv_PD_TV_f32(_a(Y), _a(lam), _a(dsa), _a(hout), _a(hinfo), _a(nsa), nd, k, maxit)
        assert rc == 1, lib.proxtv_last_error()
        assert np.array_equal(lam, scaled(case)), "the host entry did not scale the penalties in place"
        assert np.array_equal(hout, want) and np.array_equal(hinfo, info), "host entry"
        # numpy: a Fortran-ordered array of shape ns; ws a float64 ndarray, which PD_TV and PDR_TV scale in place like the reference
        w = np.array(case.ws, dtype=np.float64)
        got = front(Y.reshape(case.ns, order="F"), w, case.ds, [1] * k, max_iters=maxit)
        assert got.dtype == dt and np.array_equal(got.ravel(order="F"), want), "numpy"
        assert np.array_equal(front.last_info, info), (front.last_info, info)
        assert np.array_equal(w, scaled(case)), w
    # torch: the C-ordered tensor of the reversed shape (axis a -> nd + 1 - a) and the Fortran-ordered one of shape ns hold the
    # same memory as the flat column-major item, so the solver sees the very problem the device entry saw
    xc = Yt.reshape(case.ns[::-1])
    xf = xc.permute(tuple(range(nd - 1, -1, -1)))
    for x, ds in ((xc, [nd + 1 - d for d in case.ds]), (xf, case.ds)):
        for w in (list(case.ws), np.array(case.ws, dtype=np.float64), torch.tensor(case.ws, dtype=torch.float64)):
            got = front(x, w, ds, [1] * k, max_iters=maxit)
            assert got.shape == x.shape and got.dtype == x.dtype
            flat = got.reshape(-1) if x is xc else flat_of(got)
            assert torch.equal(flat, out), ("torch", "C" if x is xc else "F", type(w))
            assert np.array_equal(front.last_info, info)
            assert np.array_equal(np.asarray(w.cpu() if torch.is_tensor(w) else w, dtype=np.float64), case.ws), "ws was written"


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["float64", "float32"])
def test_tv1_2d_pd(ptv, port, lib, dt):
    """tv1_2d(method='pd') is PD2_TV on the terms [w, w] along axes [1, 2]: bit for bit the device entry on numpy (float64) and on a
    Fortran-ordered tensor, and within the oracle's bar."""
    case = Single("t1", "PD2", (96, 80), [1, 2], [0.2, 0.2], "noisy", 20)
    maxit = case.maxit if dt == np.float64 else F32_MAXIT
    ptv.set_engine("chunked")
    Y = case.Y(dt)
    Yt = torch.tensor(Y, device="cuda")
    out, info = dev(lib, case, Yt, maxit)
    orc, oinfo = oracle(port, case, dt, maxit)
    check_info(case, info, orc, oinfo, dt, maxit)
    assert relerr(out.double().cpu().numpy(), orc[0][0]) <= (1e-9 if dt == np.float64 else F32_BAR)
    if dt == np.float64:
        got = ptv.tv1_2d(Y.reshape(case.ns, order="F"), 0.2, max_iters=maxit, method="pd")
        assert np.array_equal(got.ravel(order="F"), out.cpu().numpy()), "numpy"
    xf = Yt.reshape(case.ns[::-1]).permute(1, 0)
    got = ptv.tv1_2d(xf, 0.2, max_iters=maxit, method="pd")
    assert got.dtype == xf.dtype and torch.equal(flat_of(got), out), "torch"


def test_every_route_was_taken():
    """Runs after the cases: the table reached every route, and the guard decided both ways."""
    if SEEN["ran64"] != len(PARAMS) or SEEN["ran32"] != len(PARAMS):
        pytest.skip("only %d + %d of %d + %d cases ran" % (SEEN["ran64"], SEEN["ran32"], len(PARAMS), len(PARAMS)))
    print("\nroutes taken: %s\nguard decisions: %s\nlargest float64 lane relerr: %.3g\nfloat32 relerr under the seq engine: %s"
          "\nfloat32 relerr, largest over the cases that took each route: %s\nfloat32 relerr per case: %s\n%d cases in %.1f s"
          % (sorted(SEEN["routes"]), sorted(SEEN["guard"]), SEEN["lane_err"], {k: "%.3g" % v for k, v in sorted(SEEN["f32_seq"].items())},
             {"%s %s" % k: "%.3g" % v for k, v in sorted(SEEN["f32_err"].items())},
             {k: "%.3g" % v for k, v in SEEN["f32_case"].items()}, 2 * len(PARAMS), time.perf_counter() - SEEN["t0"]))
    want = {"lane", "chunked", "gather-scatter", "gather-scatter-fused", "strided-direct", "gather-seq", "seq"}
    assert want <= SEEN["routes"], sorted(want - SEEN["routes"])
    assert SEEN["routes"] & {"long-tiles", "long-fallback"}, sorted(SEEN["routes"])
    assert SEEN["guard"] == {0, 1}, SEEN["guard"]
    pdr = {r for (s, r) in SEEN["f32_err"] if s == "PDR"}
    assert {"lane", "chunked", "gather-scatter", "strided-direct", "gather-seq", "seq"} <= pdr, sorted(pdr)
