"""GPU tests (-m gpu) of the batched N-D TV-L1 prox (proxtv_PD_TV_batched_* / proxtv_PD2_TV_batched_*, tvgen_batched; DESIGN.md
section 16) against the float64 oracle (orc_pd_tv / orc_pd2_tv) on every fiber route its prox passes take.

The route of a term.  Item b of shape ns is column-major; term i runs over the axis d = ds[i] - 1 and, while m items run, its pass is
one call of prox_fibers_ex (prox_dispatch.cu) on the geometry (nf m, ns[d], prod(ns[:d])) with 3 n m elements of scratch.  Case.term_route()
restates the dispatch through test_gpu_prox1d_routes.expected_route, with what differs for these calls:
  * PD_TV's passes read a plain input and may take the lane engine; PD2_TV's read x + p (IN_A_PLUS_B), which the lane engine does
    not take, so PD2_TV never does;
  * the penalty of a pass is PD_TV's ws[i] times npen (PD2_TV: ws[i]); the lane guard runs once per solve under 'auto' on the first
    2^18 of the n B input elements, with the largest of the passes' penalties;
  * strided passes always get the sparse gather / scan / scatter form, because 3 n m >= strided_scratch_elems(nf m, len) (asserted);
  * contiguous fibers too long for the chunked kernel reach the long-fiber tiles only when 3 n m >= lf_scratch_elems(nf m, len) (the
    1D entry points' 16384-sample rule does not apply here); whether the tiles' check passed is proxtv_long_fiber_last.
The lane engine needs nf m >= 1024, so a route can change while the batch solves: as items stop, m falls and a pass moves from the
lane engine to the chunked kernels.  Each case id names, per term, the route with all B items running and, after '>', the one with
only the items the cap ends still running.

What the library shows of the route: the contiguous- and strided-scan launch counters (each pass is one launch of the class of its
fibers' stride, whichever family runs it; a long-fiber pass whose tiles' check fails adds the sequential kernel), proxtv_lane_guard_last
and proxtv_long_fiber_last.  The counters cannot tell the lane kernels from the chunked ones; that distinction rests on the restatement
and the guard.

Bars, for every item b:
  * float64, every route (lane included): relerr(x_b, oracle(y_b)) <= 1e-9; info[b, 0] == the oracle's K when the stop test is
    decided by a margin (the oracle's stop value > 1e-6 (1 + 1e-9) after K - 1 iterations and <= 1e-6 (1 - 1e-9) after K; asserted
    for every item the stop rule ends), else K == maxIters (the cap ends it);
  * float32, solves the cap ends (maxIters = 8, so K is not at stake): relerr against the float64 oracle on the float32-rounded input
    <= F32_BAR = 2e-5.  The bar comes from the seq route, where every pass is the exact taut-string scan in float32: its largest
    error over these cases was 3.84e-6 on an H100 (80 GB, default power limit); the bar gives it a margin of 5x, and the seq route is
    held to a quarter of the bar so that the margin cannot erode unnoticed.  The other routes measured at most 3.84e-6 as well (the
    lane engine, which scans in double and rounds once, 2.5e-7);
  * float64 on the lane engine measured at most 2.4e-15 relative to the oracle, well inside 1e-9; the smallest stop margin of the
    table was 1.15 % (the oracle's stop value after K - 1 or K iterations against 1e-6);
  * under seq, chunked and chunked-strided: each item bit for bit the single-item proxtv_PD*_TV_dev_* with the same info row, and the
    recorded forward bit for bit the no-grad one with the tape's K table == info[:, 0];
  * the batched dev entry on the current stream and on a side stream, the host entry, tvgen_batched on a C-ordered and on an
    item-column-major tensor; the penalty arrays come back unmodified.
"""
import ctypes as C
import time

import numpy as np
import pytest

from conftest import relerr
from test_gpu_pd_batched import item
from test_gpu_prox1d_routes import LF_TL, LF_W, chunked_contig_ok, expected_route, guard_ok

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

STOP_PD = 1e-6                      # ptv_internal.h / the oracle's ORC_STOP_PD
STOP_MARGIN = 1e-9                  # the stop value's distance from STOP_PD, relative, that decides K on both sides
F32_MAXIT = 8
F32_BAR = 2e-5                      # float32 relerr against the oracle: 5x the largest seen on the seq route (module docstring)
ENGINES = ("seq", "chunked", "chunked-strided", "lane", "auto")
EXACT_ENGINES = ("seq", "chunked", "chunked-strided")
KC_CONTIG, KC_STRIDED = 0, 1


def strided_scratch_elems(nf, ln):
    """prox_dispatch.cu: elements the sparse form of a strided pass needs."""
    return 2 * nf * ln + 2 * nf * (-(-ln // 32)) + 64


def lf_scratch_elems(nf, ln):
    """long_fiber.cu: elements the long-fiber tiles need."""
    return 2 * nf * (-(-ln // LF_TL)) * LF_W + 8


# ---- the items ---------------------------------------------------------------------------------------------------------------
def make_item(kind, ns, seed):
    """One flat column-major item: item()'s 'const', 'smooth' and 'noisy', and 'smooth~s', 'smooth' plus N(0, s) noise, which stops
    later the larger s is."""
    if kind.startswith("smooth~"):
        s = float(kind[7:])
        return item("smooth", ns, seed) + np.random.default_rng(1000 + seed).normal(0, s, int(np.prod(ns)))
    return item(kind, ns, seed)


class Case:
    def __init__(self, key, pd2, ns, ds, ws, kinds, maxit, engines=ENGINES):
        self.key, self.pd2, self.ns, self.ds, self.ws, self.kinds, self.maxit = key, pd2, tuple(ns), list(ds), list(ws), kinds, maxit
        self.engines = engines
        self.B, self.n = len(kinds), int(np.prod(ns))

    def Y(self, dt):
        return np.concatenate([make_item(k, self.ns, 11 * b + 3) for b, k in enumerate(self.kinds)]).astype(dt)

    def lam(self, i, dt):
        """The penalty of term i's passes, in the storage type."""
        return float(np.asarray(self.ws[i] * (1 if self.pd2 else len(self.ws)), dtype=dt))

    def guard(self, dt):
        """(decision, margin) of the lane guard for this input (the auto engine consults it once per solve)."""
        key = (self.key, np.dtype(dt).name)
        if key not in _GUARD:
            _GUARD[key] = guard_ok(self.Y(dt), max(self.ws) * (1 if self.pd2 else len(self.ws)))
        return _GUARD[key]

    def term_route(self, i, m, dt, engine, guard=None):
        ns, d = self.ns, self.ds[i] - 1
        ln, inc = ns[d], int(np.prod(ns[:d]))
        nf = self.n // ln * m
        isz = np.dtype(dt).itemsize
        if guard is None:
            guard = self.guard(dt)[0]
        eng = engine
        if self.pd2 and engine in ("lane", "auto"):
            eng = "chunked"                                       # IN_A_PLUS_B: the lane engine is never asked
        r = expected_route(dt, False, nf, ln, inc, eng, self.lam(i, dt), guard)
        if r in ("gather-scatter", "gather-seq"):
            assert 3 * self.n * m >= strided_scratch_elems(nf, ln), "the strided pass would take the dense form"
        if inc == 1 and eng != "seq" and ln >= 64 and not chunked_contig_ok(isz, False, nf, ln):
            tiles = ln >= 2 * LF_W and nf * (-(-ln // LF_TL)) <= 65535 and 3 * self.n * m >= lf_scratch_elems(nf, ln)
            r = "long-tiles" if tiles else "seq"
        return r

    def final_m(self):
        """Items running in the last iteration by the case's design: the ones the cap ends (one term: every item, at K = 1 or 2)."""
        if len(self.ws) == 1:
            return self.B
        return sum(k == "noisy" for k in self.kinds)

    def id(self, engine, dt):
        parts = []
        for i in range(len(self.ws)):
            a, b = self.term_route(i, self.B, dt, engine), self.term_route(i, max(self.final_m(), 1), dt, engine)
            parts.append("%d:%s" % (self.ds[i], a if a == b else a + ">" + b))
        return "%s-%s-%s-%s-B%d-%s-%s" % (self.key, "PD2" if self.pd2 else "PD", np.dtype(dt).name, "x".join(map(str, self.ns)),
                                          self.B, engine, "+".join(parts))


CASES = [
    # chunked (axis 1, 80 m fibers) and the sparse gather / scatter (axis 2, inc 96); the direct strided kernel under chunked-strided
    Case("c1", False, (96, 80), [1, 2], [0.2, 0.25], ["noisy", "const", "smooth", "smooth~0.05", "smooth~0.02"], 60),
    # 1536 m fibers on axes 1 and 2: the lane engine at every m (contiguous and strided); axis 3 is shorter than 64: sequential
    Case("c2", False, (64, 64, 24), [1, 2, 3], [0.1, 0.1, 0.1], ["noisy", "smooth~0.02", "const"], 40),
    # the engine changes mid-solve: axis 1 is on the lane engine while >= 13 items run, axis 2 while >= 8; four constant items
    # stop at K = 2, the smooth ones at K = 15 .. 50, the noisy ones run to the cap
    Case("c3", False, (128, 80), [1, 2], [0.2, 0.25],
         ["const", "noisy", "smooth", "const", "smooth~0.02", "smooth~0.1", "const", "smooth~0.05", "noisy", "smooth~0.02",
          "smooth", "const", "smooth~0.05", "smooth~0.1", "noisy", "smooth~0.02"], 60),
    # row pitch 129 * 8 = 1032 bytes (129 * 4 = 516), not a multiple of 16: the lane engine refuses both axes though nf m >= 1024;
    # axis 1 repeated; inc 129 is odd: no direct strided kernel, the gather / scatter under every engine but seq
    Case("c4", False, (129, 70), [1, 2, 1], [0.1, 0.15, 0.1],
         ["smooth~0.02", "noisy", "const", "smooth", "smooth~0.05", "noisy", "smooth~0.02", "const",
          "smooth", "noisy", "smooth~0.05", "const", "smooth~0.02", "noisy", "smooth", "const"], 30),
    # PD2_TV: the fused x + p input through the chunked contiguous kernel and the sparse gather / scatter
    Case("c5", True, (96, 80), [1, 2], [0.2, 0.25], ["noisy", "const", "smooth", "smooth~0.05", "smooth~0.02"], 20),
    # PD2_TV: the fused input on a strided axis shorter than 64 (sequential) and on a contiguous one (chunked)
    Case("c6", True, (70, 66, 9), [3, 1], [0.2, 0.3], ["noisy", "smooth~0.02", "const", "smooth"], 20),
    # strided fibers longer than the chunked kernel takes (22326 float64, 32768 float32 samples): gathered, then sequential
    Case("c7", False, (2, 33000), [2], [0.3], ["noisy", "smooth~0.05"], 20),
    # one contiguous fiber per item, longer than the chunked kernel takes: the long-fiber tiles (3 n m >= lf_scratch_elems)
    Case("c8", False, (40000,), [1], [0.3], ["noisy", "smooth~0.05"], 20),
    # the guard's other decision: penalties above the mean step of c2's input (the lane route otherwise)
    Case("c2hi", False, (64, 64, 24), [1, 2, 3], [1.0, 1.0, 1.0], ["noisy", "smooth~0.02", "const"], 40, engines=("auto",)),
]
CASE_BY_KEY = {c.key: c for c in CASES}
PARAMS = [(c, e) for c in CASES for e in c.engines]
_GUARD = {}
SEEN = {"routes": set(), "switch": set(), "guard": set(), "ran64": 0, "ran32": 0, "t0": None, "f32_err": {}, "lane_err": 0.0,
        "margin": 1.0}
IDS64 = [c.id(e, np.float64) for c, e in PARAMS]
IDS32 = [c.id(e, np.float32) for c, e in PARAMS]


# ---- the oracle, once per case, dtype and cap ---------------------------------------------------------------------------------
_ORACLE = {}


def oracle(port, case, dt, maxit):
    """Per item: (x in float64, flat; K; stop after K; stop after K - 1, or inf when K == 1).  float32: the float64 oracle on the
    float32-rounded input."""
    key = (case.key, np.dtype(dt).name, maxit)
    if key not in _ORACLE:
        fn = port.pd2_tv if case.pd2 else port.pd_tv
        Y = case.Y(dt).astype(np.float64)
        rows = []
        for b in range(case.B):
            V = Y[b * case.n:(b + 1) * case.n].reshape(case.ns, order="F")
            x, info = fn(V, list(case.ws), case.ds, maxit=maxit)
            K = int(info[0])
            prev = fn(V, list(case.ws), case.ds, maxit=K - 1)[1][1] if K > 1 else np.inf
            rows.append((x.ravel(order="F"), K, float(info[1]), float(prev)))
        _ORACLE[key] = rows
    return _ORACLE[key]


# ---- calls ----------------------------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr())


def _a(a):
    return C.c_void_p(a.ctypes.data)


def sfx(dt):
    return "f32" if dt in (np.float32, torch.float32) else "f64"


def solver(case):
    return "PD2_TV" if case.pd2 else "PD_TV"


def batched_dev(lib, case, Yt, maxit, stream=None, record=False):
    """proxtv_PD*_TV_batched_dev_* (or _record_dev_*) on the flat tensor Yt; (out, info (B, 3), tape or None)."""
    lam, dsa, nsa = np.array(case.ws, dtype=np.float64), np.array(case.ds, dtype=np.float64), np.array(case.ns, dtype=np.int32)
    out = torch.full_like(Yt, float("nan"))
    info = np.zeros(3 * case.B)
    args = [_p(Yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(case.ns), len(case.ws), case.B, maxit]
    tape = None
    if record:
        nb = getattr(lib, "proxtv_%s_batched_tape_bytes" % solver(case))(_a(nsa), len(case.ns), len(case.ws), case.B, maxit)
        tape = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        args += [_p(tape), nb]
    f = getattr(lib, "proxtv_%s_batched_%sdev_%s" % (solver(case), "record_" if record else "", sfx(Yt.dtype)))
    if stream is None:
        assert f(*args, C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 1, lib.proxtv_last_error()
    else:
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            assert f(*args, C.c_void_p(stream.cuda_stream)) == 1, lib.proxtv_last_error()
        stream.synchronize()
    assert np.array_equal(lam, np.array(case.ws, dtype=np.float64)), "the penalties were written"
    return out, info.reshape(case.B, 3), tape


def single_dev(lib, case, yt, maxit):
    lam, dsa, nsa = np.array(case.ws, dtype=np.float64), np.array(case.ds, dtype=np.float64), np.array(case.ns, dtype=np.int32)
    out = torch.full_like(yt, float("nan"))
    info = np.zeros(3)
    f = getattr(lib, "proxtv_%s_dev_%s" % (solver(case), sfx(yt.dtype)))
    assert f(_p(yt), _a(lam), _a(dsa), _p(out), _a(info), _a(nsa), len(case.ns), len(case.ws), maxit,
             C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 1, lib.proxtv_last_error()
    return out, info


def reset_long_fiber_hook(lib):
    """Any 1D prox call clears proxtv_long_fiber_last to -1 (the batched N-D entries leave it as their last pass set it)."""
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    y = torch.empty_like(x)
    assert lib.proxtv_prox_fibers_dev_f64(_p(x), _p(y), 1, 8, 1, C.c_double(0.5), None, None) == 1
    assert lib.proxtv_long_fiber_last() == -1


def counters(lib):
    ms, launches, spans = (C.c_double * 3)(), (C.c_longlong * 3)(), (C.c_longlong * 3)()
    lib.proxtv_profile_read(ms, launches, spans)
    return list(launches)


@pytest.fixture
def lib(ptv):
    L = ptv.load()
    prev = ptv.set_engine("auto")
    yield L
    ptv.set_engine(prev)
    L.proxtv_profile_reset()


# ---- checks -------------------------------------------------------------------------------------------------------------------
def routes_taken(case, dt, engine, K, guard):
    """[(term, iteration j, m_j, route)] from the K table: iteration j runs the items with K_b >= j."""
    out = []
    for j in range(1, int(K.max()) + 1):
        m = int((K >= j).sum())
        for i in range(len(case.ws)):
            out.append((i, j, m, case.term_route(i, m, dt, engine, guard)))
    return out


def check_routes(lib, case, dt, engine, info, launches, guard):
    """The launch counters and the long-fiber hook against the restated routes; returns the routes taken, long ones resolved."""
    K = info[:, 0].astype(int)
    taken = routes_taken(case, dt, engine, K, guard)
    strided = [int(np.prod(case.ns[:case.ds[i] - 1])) > 1 for i in range(len(case.ws))]
    want = [sum(1 for i, _, _, _ in taken if not strided[i]), sum(1 for i, _, _, _ in taken if strided[i])]
    long_passes = sum(1 for _, _, _, r in taken if r == "long-tiles")
    hook = lib.proxtv_long_fiber_last()
    assert launches[KC_STRIDED] == want[1], ("strided launches", launches, want)
    if long_passes:
        assert hook in (0, 1), hook
        extra = launches[KC_CONTIG] - want[0]                     # one sequential launch per pass whose tiles' check failed
        assert 0 <= extra <= long_passes and (hook == 1 or extra >= 1), ("contiguous launches", launches, want, hook)
    else:
        assert hook == -1, hook
        assert launches[KC_CONTIG] == want[0], ("contiguous launches", launches, want)
    names = set()
    for i, _, _, r in taken:
        if r == "long-tiles":
            r = "long-tiles" if hook == 1 else "long-fallback"
        if r == "gather-scatter" and case.pd2:
            r = "gather-scatter-fused"
        names.add(r)
        if r == "strided-direct":
            assert engine == "chunked-strided"
    for i in range(len(case.ws)):
        seq_i = [r for t, _, _, r in taken if t == i]
        if seq_i[0] == "lane" and seq_i[-1] != "lane":
            SEEN["switch"].add(case.key)
    return names


def check_K(case, info, orc, dt, maxit):
    """info[b, 0] == the oracle's K for every item.  Where the stop rule ends an item (K < maxIters), the oracle's stop values must
    decide it by a margin on both sides of the threshold: 1e-9 in float64; 1e-2 in float32, whose stop values differ from the
    oracle's by more (under the cap of 8 the rule ends only constant items, stop value 0, and one smooth PD2_TV item, 3 % above)."""
    margin_req = STOP_MARGIN if dt == np.float64 else 1e-2
    for b, (_, K, stop, prev) in enumerate(orc):
        if K < maxit:
            assert prev > STOP_PD * (1 + margin_req) and stop <= STOP_PD * (1 - margin_req), \
                ("the stop test of item %d is not decided by a margin" % b, prev, stop)
            SEEN["margin"] = min(SEEN["margin"], prev / STOP_PD - 1, 1 - stop / STOP_PD)
        assert int(info[b, 0]) == K, ("K", b, info[:, 0], [o[1] for o in orc])


def check_values(case, out, orc, dt, bar):
    got = out.double().cpu().numpy()
    worst = 0.0
    for b, (x, _, _, _) in enumerate(orc):
        e = relerr(got[b * case.n:(b + 1) * case.n], x)
        assert e <= bar, ("item", b, e, bar)
        worst = max(worst, e)
    return worst


def check_consistency(lib, case, Yt, out, info, maxit):
    """seq / chunked / chunked-strided: every item is the single-item solve bit for bit, and the recorded forward is the no-grad one."""
    n = case.n
    for b in range(case.B):
        ref, rinfo = single_dev(lib, case, Yt[b * n:(b + 1) * n].clone(), maxit)
        assert torch.equal(out[b * n:(b + 1) * n], ref) and np.array_equal(info[b], rinfo), ("single item", b, info[b], rinfo)
    rout, rinfo, tape = batched_dev(lib, case, Yt, maxit, record=True)
    assert torch.equal(rout, out) and np.array_equal(rinfo, info), "recorded forward"
    assert np.array_equal(tape[256:256 + 4 * case.B].cpu().numpy().view(np.int32), info[:, 0].astype(np.int32)), "tape K table"


def run_case(ptv, port, lib, case, engine, dt):
    maxit = case.maxit if dt == np.float64 else F32_MAXIT
    Y = case.Y(dt)
    guard, gmargin = case.guard(dt)
    if engine == "auto":
        assert gmargin > 1e-6, "the data sits on the lane guard's threshold"
    orc = oracle(port, case, dt, maxit)
    Yt = torch.tensor(Y, device="cuda")
    ptv.set_engine(engine)
    reset_long_fiber_hook(lib)
    lib.proxtv_profile_reset()
    out, info, _ = batched_dev(lib, case, Yt, maxit)
    launches = counters(lib)
    if engine == "auto":
        assert lib.proxtv_lane_guard_last() == int(guard), (lib.proxtv_lane_guard_last(), guard)
        SEEN["guard"].add(int(guard))
    check_K(case, info, orc, dt, maxit)
    names = check_routes(lib, case, dt, engine, info, launches, guard)
    assert len(case.ws) == 1 or np.all(info[:, 0][np.array([k == "noisy" for k in case.kinds])] == maxit), info
    return Yt, out, info, orc, names, maxit


@pytest.mark.parametrize("case,engine", PARAMS, ids=IDS64)
def test_forward_f64(ptv, port, lib, case, engine):
    if SEEN["t0"] is None:
        SEEN["t0"] = time.perf_counter()
    Yt, out, info, orc, names, maxit = run_case(ptv, port, lib, case, engine, np.float64)
    err = check_values(case, out, orc, np.float64, 1e-9)
    if any(r == "lane" for r in names):
        SEEN["lane_err"] = max(SEEN["lane_err"], err)
    if engine in EXACT_ENGINES:
        check_consistency(lib, case, Yt, out, info, maxit)
    if engine == "chunked":                                       # the same solve on a side stream
        sout, sinfo, _ = batched_dev(lib, case, Yt, maxit, stream=torch.cuda.Stream())
        assert torch.equal(sout, out) and np.array_equal(sinfo, info), "side stream"
    SEEN["routes"] |= names
    SEEN["ran64"] += 1


@pytest.mark.parametrize("case,engine", PARAMS, ids=IDS32)
def test_forward_f32(ptv, port, lib, case, engine):
    Yt, out, info, orc, names, maxit = run_case(ptv, port, lib, case, engine, np.float32)
    err = check_values(case, out, orc, np.float32, F32_BAR)
    if engine == "seq":
        assert err <= F32_BAR / 4, ("the float32 bar no longer has its margin over the seq route", err)
    for r in names:
        SEEN["f32_err"][r] = max(SEEN["f32_err"].get(r, 0.0), err)
    if engine in EXACT_ENGINES:
        check_consistency(lib, case, Yt, out, info, maxit)
    SEEN["ran32"] += 1


# ---- the other entry points ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["c1", "c5", "c6"])
def test_host_entry(ptv, port, lib, key):
    """proxtv_PD*_TV_batched_f64 / _f32 on host arrays: bit for bit the device entry, and within the bars of the oracle."""
    case = CASE_BY_KEY[key]
    ptv.set_engine("chunked")
    for dt in (np.float64, np.float32):
        maxit = case.maxit if dt == np.float64 else F32_MAXIT
        Y = case.Y(dt)
        lam, dsa, nsa = np.array(case.ws), np.array(case.ds, dtype=np.float64), np.array(case.ns, dtype=np.int32)
        out = np.full_like(Y, np.nan)
        info = np.zeros(3 * case.B)
        f = getattr(lib, "proxtv_%s_batched_%s" % (solver(case), sfx(dt)))
        assert f(_a(Y), _a(lam), _a(dsa), _a(out), _a(info), _a(nsa), len(case.ns), len(case.ws), case.B, maxit) == 1, \
            lib.proxtv_last_error()
        assert np.array_equal(lam, case.ws)
        dout, dinfo, _ = batched_dev(lib, case, torch.tensor(Y, device="cuda"), maxit)
        assert np.array_equal(out, dout.cpu().numpy()) and np.array_equal(info.reshape(case.B, 3), dinfo)
        orc = oracle(port, case, dt, maxit)
        check_K(case, dinfo, orc, dt, maxit)
        check_values(case, dout, orc, dt, 1e-9 if dt == np.float64 else F32_BAR)


@pytest.mark.parametrize("key", ["c2", "c5", "c6"])
@pytest.mark.parametrize("engine", ["chunked", "auto"])
def test_tvgen_batched_layouts(ptv, port, lib, key, engine):
    """tvgen_batched on a C-ordered tensor (item b is the array of shape ns, stored in C order: the solver sees the column-major array
    of the reversed shape and axis a becomes nds + 1 - a) and on an item-column-major one (the flat layout of the C ABI), against the
    oracle on the item of shape ns; ws as a list and as an ndarray, never written."""
    case = CASE_BY_KEY[key]
    ptv.set_engine(engine)
    nd = len(case.ns)
    perm = (0,) + tuple(range(nd, 0, -1))
    for dt in (np.float64, np.float32):
        maxit = case.maxit if dt == np.float64 else F32_MAXIT
        Y = case.Y(dt)
        items = np.ascontiguousarray(np.stack([Y[b * case.n:(b + 1) * case.n].reshape(case.ns, order="F") for b in range(case.B)]))
        orc = oracle(port, case, dt, maxit)
        bar = 1e-9 if dt == np.float64 else F32_BAR
        xc = torch.tensor(items, device="cuda")                                  # C order
        xf = xc.permute(perm).contiguous().permute(perm)                         # items column-major, batch slowest
        assert xc.is_contiguous() and not xf.is_contiguous()
        for x in (xc, xf):
            for w in (list(case.ws), np.array(case.ws)):
                got = ptv.tvgen_batched(x, w, case.ds, [1] * len(case.ws), max_iters=maxit)
                assert got.shape == x.shape and got.stride() == x.stride()
                assert list(w) == case.ws
                info = ptv.tvgen_batched.last_info
                check_K(case, info, orc, dt, maxit)
                flat = torch.cat([got[b].permute(tuple(range(nd - 1, -1, -1))).reshape(-1) for b in range(case.B)])
                check_values(case, flat, orc, dt, bar)
        if engine == "chunked":                                   # column-major items are the C ABI's layout: the same bits
            want, _, _ = batched_dev(lib, case, torch.tensor(Y, device="cuda"), maxit)
            got = ptv.tvgen_batched(xf, case.ws, case.ds, [1] * len(case.ws), max_iters=maxit)
            flat = torch.cat([got[b].permute(tuple(range(nd - 1, -1, -1))).reshape(-1) for b in range(case.B)])
            assert torch.equal(flat, want)


def test_every_route_was_taken():
    """Runs after the cases: the table reached every route, one case switched from the lane engine to the chunked kernels during
    its solve, and the guard decided both ways."""
    if SEEN["ran64"] != len(PARAMS) or SEEN["ran32"] != len(PARAMS):
        pytest.skip("only %d + %d of %d + %d cases ran" % (SEEN["ran64"], SEEN["ran32"], len(PARAMS), len(PARAMS)))
    print("\nroutes taken: %s\nlane -> chunked during the solve: %s\nguard decisions: %s\nlargest float64 lane relerr: %.3g"
          "\nsmallest stop margin: %.3g\nfloat32 relerr, largest over the cases that took each route: %s\n%d cases in %.1f s"
          % (sorted(SEEN["routes"]), sorted(SEEN["switch"]), sorted(SEEN["guard"]), SEEN["lane_err"], SEEN["margin"],
             {k: "%.3g" % v for k, v in sorted(SEEN["f32_err"].items())}, 2 * len(PARAMS), time.perf_counter() - SEEN["t0"]))
    want = {"lane", "chunked", "gather-scatter", "gather-scatter-fused", "strided-direct", "gather-seq", "seq"}
    assert want <= SEEN["routes"], sorted(want - SEEN["routes"])
    assert SEEN["routes"] & {"long-tiles", "long-fallback"}, sorted(SEEN["routes"])
    assert SEEN["switch"], "no case moved from the lane engine to the chunked kernels during its solve"
    assert SEEN["guard"] == {0, 1}, SEEN["guard"]
