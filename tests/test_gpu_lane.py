"""GPU tests (-m gpu) of the lane-per-fiber engine's CUDA kernels (kernels_lane.cu), held to a BIT-EXACT bar.

The lane engine's output is a pure function of its input: whatever the window, the epoch length, the chunking, the halo or the repairs,
every fiber equals the plain sequential slope-form scan of that fiber (`slope_seq`, lane_core.cuh), float64 as it is and float32
storage scanned in double and rounded once (pinned on the CPU by
test_lane_emulation.py::test_lane_output_is_the_sequential_scan_bit_for_bit).  The host reference here is that scan
(tests/emu/emu_lane.cu: emu_slope_fibers_*, loaded by tests/lane_emu.py), so these tests check what only the device runs: the scan loop's device copy (run_dev),
the TMA feeds (strided tiles, swizzled contiguous boxes, staged operand tiles), the three drains (direct, boxed TMA store, transposed
exchange), the repair path's shared-memory staging, the group counters that pick the verifying warp, and the task plan as the device
sizes it.  Bars:
  * every op, dtype, layout, shape, tuning variant and chunking: np.array_equal with the host reference (op arithmetic in numpy, in
    the storage type, with the association of PassOp);
  * op 0 in float64 also against the oracle port's taut string: <= 1e-9 relative, identical jump sets;
  * whole DR2_TV solves on the lane engine (numpy, torch row- and column-major, batched, float64 / float32): bit for bit against a
    host driver with the schedule of solver.cu on inputs on a dyadic grid (integers / 256, so that the start value 2 * mean is exact
    in any summation order).
"""
import ctypes as C
import subprocess
import sys

import numpy as np
import pytest

import lane_emu
from conftest import ROOT, jumps, relerr
from lane_emu import slope_fibers
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emu():
    return lane_emu.load()

DEFAULT_TUNING = (0, 32, -1)          # chunk length (0: as many chunks as fill one wave), halo rows, variant (-1: per storage type)
LENS = (2, 3, 7, 8, 9, 16, 17, 33, 64, 65, 128, 257, 1000, 4096)
VARIANTS = (0, 1, 5, 6, 7)
# (data kind, lambda), cycled through the shapes of a grid in a fixed order
CASES = (("blocks", 0.2), ("ties", 1.0), ("const", 0.5), ("ramp", 5.0), ("alt", 0.3), ("plateau", 0.5), ("offset", 0.2),
         ("blocks", 1e-12), ("ties", 1e4), ("blocks", 2.0))


@pytest.fixture
def lane_lib(ptv):
    """The raw C ABI with the lane engine's default tuning, restored after the test whatever it set."""
    lib = ptv.load()
    lib.proxtv_lane_tuning(*DEFAULT_TUNING)
    yield lib
    lib.proxtv_lane_tuning(*DEFAULT_TUNING)


@pytest.fixture
def engine(ptv):
    """Sets the 2D engine for the test (call it with a name) and restores the previous one afterwards."""
    prev = ptv.set_engine("auto")
    ptv.set_engine(prev)
    yield ptv.set_engine
    ptv.set_engine(prev)


def make(kind, nf, ln, rng):
    """(nf, ln) fibers of one data kind (float64)."""
    if kind == "blocks":                                     # cfg-2 style: piecewise constant blocks + noise
        return np.repeat(rng.normal(0, 1, (nf, ln // 16 + 1)), 16, axis=1)[:, :ln] + rng.normal(0, 0.3, (nf, ln))
    if kind == "ties":                                       # integer values: exact ties everywhere
        return np.round(rng.normal(0, 3, (nf, ln)))
    if kind == "const":
        return np.full((nf, ln), 2.5)
    if kind == "ramp":
        return np.tile(np.linspace(-3, 3, ln), (nf, 1)) + rng.normal(0, 0.01, (nf, 1))
    if kind == "alt":
        return np.where(np.arange(ln) % 2 == 0, 1.0, -1.0)[None, :] * np.ones((nf, 1))
    if kind == "plateau":
        a = rng.normal(0, 1, (nf, ln)); a[:, ln // 3:2 * ln // 3] = 0.3; return a
    if kind == "offset":
        return 1e6 + rng.normal(0, 1, (nf, ln))
    raise ValueError(kind)


def layout(F, inc):
    """Flat array holding the fibers F (nf, ln) under the slicing rule (nf, ln, inc): contiguous fibers (inc == 1), or slabs of inc
    adjacent fibers (element r of fiber s * inc + c at s * inc * ln + r * inc + c)."""
    nf, ln = F.shape
    if inc == 1:
        return np.ascontiguousarray(F).ravel()
    return np.ascontiguousarray(F.reshape(nf // inc, inc, ln).transpose(0, 2, 1)).ravel()


def fiber_major(v, nf, ln, inc):
    """A flat array in the (nf, ln, inc) layout rewritten fiber-major (element r of fiber f at f * ln + r): the transposed ops' output."""
    return v.copy() if inc == 1 else np.ascontiguousarray(v.reshape(nf // inc, ln, inc).transpose(0, 2, 1)).ravel()


def expected(emu, op, A, B, Cc, nf, ln, inc, lam):
    """Host reference of one lane pass: the op's input arithmetic, the sequential scan of every fiber, the op's output arithmetic --
    in the storage type, with the association of PassOp (kernels_lane.cu); transposed ops (3-6) return fiber-major arrays."""
    T = A.dtype.type
    if op == 1:
        d = Cc - B; a = A - (T(2) * d - Cc)
    elif op == 2:
        a = A - (Cc - B)
    else:
        a = A
    x = slope_fibers(emu, a, nf, ln, inc, lam)
    x2 = None
    if op == 1:
        x1 = (Cc - B) + x
    elif op == 3:
        d = Cc - x; x2 = d; x1 = B - (T(2) * d - Cc)
    elif op == 4:
        x1 = B - (Cc - x)
    elif op == 5:
        x1 = B + x
    else:
        x1 = x
    if op >= 3:
        x1 = fiber_major(x1, nf, ln, inc)
        x2 = None if x2 is None else fiber_major(x2, nf, ln, inc)
    return x1, x2


def run_lane(lib, op, A, B, Cc, nf, ln, inc, lam):
    """One lane pass on the GPU through proxtv_lane_prox(2)_dev_*; returns (ok, X, X2) as numpy arrays."""
    import torch
    dev = torch.device("cuda")
    t = lambda a: None if a is None else torch.from_numpy(a).to(dev)          # noqa: E731
    tA, tB, tC = t(A), t(B), t(Cc)
    X = torch.full((A.size,), float("nan"), dtype=tA.dtype, device=dev)
    X2 = torch.full((A.size,), float("nan"), dtype=tA.dtype, device=dev) if op == 3 else None
    p = lambda a: None if a is None else C.c_void_p(a.data_ptr())              # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if op == 3:
        ok = lib.proxtv_lane_prox2_dev_f64(op, p(tA), p(tB), p(tC), p(X), p(X2), nf, ln, inc, float(lam), st)
    elif A.dtype == np.float32:
        ok = lib.proxtv_lane_prox_dev_f32(op, p(tA), p(tB), p(tC), p(X), nf, ln, inc, float(lam), st)
    else:
        ok = lib.proxtv_lane_prox_dev_f64(op, p(tA), p(tB), p(tC), p(X), nf, ln, inc, float(lam), st)
    torch.cuda.synchronize()
    return ok, X.cpu().numpy(), None if X2 is None else X2.cpu().numpy()


def first_diff(got, want, nf, ln, inc, fmajor):
    """(fiber, row) of the first differing element, for the failure message."""
    bad = np.nonzero(~((got == want) | (np.isnan(got) & np.isnan(want))))[0]
    if bad.size == 0:
        return None
    e = int(bad[0])
    if fmajor or inc == 1:
        return e // ln, e % ln
    s, rem = divmod(e, inc * ln)
    return s * inc + rem % inc, rem // inc


def check_op(emu, lib, op, F, nf, ln, inc, lam, dt, rng, what):
    """Lay out the fibers F, run op `op`, compare bit for bit; returns the device result of X (in its own layout)."""
    T = np.dtype(dt).type
    A = layout(F, inc).astype(dt)
    B = rng.normal(0, 1, A.size).astype(dt) if op in (1, 2, 3, 4, 5) else None
    Cc = rng.normal(0, 1, A.size).astype(dt) if op in (1, 2, 3, 4) else None
    lam = T(lam)
    ok, X, X2 = run_lane(lib, op, A, B, Cc, nf, ln, inc, lam)
    assert ok == 1, (what, op, lib.proxtv_last_error())
    w1, w2 = expected(emu, op, A, B, Cc, nf, ln, inc, lam)
    assert np.array_equal(X, w1), (what, "op", op, "first differing (fiber, row)", first_diff(X, w1, nf, ln, inc, op >= 3))
    if w2 is not None:
        assert np.array_equal(X2, w2), (what, "op", op, "X2: first differing (fiber, row)", first_diff(X2, w2, nf, ln, inc, True))
    return A, X


def admitted(ln, inc, dt, transposed):
    """The lane engine's pitch rule: the row pitch (CONTIG: a fiber, STRIDED: a slab row) and, for transposed results, a fiber of the
    output must be multiples of 16 bytes."""
    es = np.dtype(dt).itemsize
    pitch = (ln if inc == 1 else inc) * es
    return pitch % 16 == 0 and (not transposed or ln * es % 16 == 0)


def ops_for(inc, dt):
    if inc == 1:
        return (0,)
    return (0, 1, 2, 3, 4, 5, 6) if dt == np.float64 else (0, 1, 2, 4, 5, 6)     # op 3 has a float64 entry point only


# (nf, inc): contiguous fibers with partial last groups; one slab (a single group / a partial group); many slabs (a batch or the 2nd
# and 3rd dimensions of a volume) with inc = 36, not a multiple of 32
GEOMS = ((33, 1), (100, 1), (32, 32), (100, 100), (108, 36))


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_ops_layouts_shapes_bit_exact(emu, lane_lib, port, dt):
    """Every op on every admitted (layout, len) of the grid, default tuning, data kinds and lambdas cycled through the shapes."""
    rng = np.random.default_rng(101)
    k = 0
    ran = 0
    for nf, inc in GEOMS:
        for ln in LENS:
            for op in ops_for(inc, dt):
                if not admitted(ln, inc, dt, op >= 3):
                    continue
                kind, lam = CASES[k % len(CASES)]; k += 1
                F = make(kind, nf, ln, rng)
                A, X = check_op(emu, lane_lib, op, F, nf, ln, inc, lam, dt, rng, (nf, ln, inc, kind, lam))
                ran += 1
                if op == 0 and dt == np.float64:          # the slope form against the reference's own taut string
                    for j in range(0, nf, 7):
                        idx = (np.arange(ln) + j * ln) if inc == 1 else ((j // inc) * inc * ln + j % inc + np.arange(ln) * inc)
                        want = port.tv1_linearized(A[idx], lam)
                        assert np.abs(X[idx] - want).max() <= 1e-9 * max(1.0, np.abs(want).max()), (nf, ln, inc, kind, lam, j)
                        assert np.array_equal(jumps(X[idx], 1e-9), jumps(want, 1e-9)), (nf, ln, inc, kind, lam, j)
    assert ran >= (130 if dt == np.float64 else 110)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_pd_geometry_bit_exact(emu, lane_lib, dt):
    """The geometry of the ND Dykstra / parallel DR solvers: >= 1024 fibers of >= 64 samples (more groups than one wave needs chunks)."""
    rng = np.random.default_rng(102)
    for nf, ln, inc, ops in ((1024, 64, 1, (0,)), (2048, 128, 1024, (0, 5)), (4096, 96, 2048, (0,))):
        for op in ops:
            check_op(emu, lane_lib, op, make("blocks", nf, ln, rng), nf, ln, inc, 0.2, dt, rng, ("pd", nf, ln, inc))


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_variants_and_chunkings_bit_exact(emu, lane_lib, dt):
    """Every tuning variant (window rows x warps per CTA x epoch length; float32 variant 0 is the 64-row window, not its default) with
    the default plan, forced chunk lengths and halo 0 (every chunk boundary is repaired): the same bits as the sequential scan."""
    rng = np.random.default_rng(103)
    F1000 = make("blocks", 108, 1000, rng); F257 = make("plateau", 108, 257, rng); Fc = make("blocks", 100, 1000, rng)
    for variant in VARIANTS:
        for clen, halo in ((0, 32), (64, 32), (128, 32), (0, 0), (64, 0)):
            lane_lib.proxtv_lane_tuning(clen, halo, variant)
            lane_lib.proxtv_lane_stats(1)
            what = ("variant", variant, "clen", clen, "halo", halo)
            check_op(emu, lane_lib, 0, Fc, 100, 1000, 1, 0.2, dt, rng, what + ("contig",))
            check_op(emu, lane_lib, 0, F257, 108, 257, 36, 0.5, dt, rng, what + ("strided 257",))
            for op in ops_for(36, dt):
                check_op(emu, lane_lib, op, F1000, 108, 1000, 36, 0.2, dt, rng, what + ("strided",))
            reps = lane_lib.proxtv_lane_stats(1)
            if halo == 0:
                assert reps > 0, what                    # cold starts right at the boundaries: the repair path did the work
            print("REPAIRS %s variant=%d clen=%d halo=%d: %d" % (np.dtype(dt).name, variant, clen, halo, reps))


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_repair_path_bit_exact(emu, lane_lib, dt):
    """Cases built to need the repair path -- halo 0 with chunks, lambda = 1e4 (one segment per fiber: lanes retire), constant fibers
    longer than the 256 rows the repair stages at a time (the stage refills) -- each must have repaired (> 0) and be bit-exact."""
    rng = np.random.default_rng(104)
    cases = (("halo 0", (64, 0), "blocks", 0.2, 100, 1000, 1, (0,)),
             ("halo 0 strided", (64, 0), "blocks", 0.2, 108, 1000, 36, (0, 1, 5)),
             ("lambda 1e4", DEFAULT_TUNING[:2], "blocks", 1e4, 100, 1000, 100, (0, 2, 4)),
             ("lambda 1e4 contig", DEFAULT_TUNING[:2], "ties", 1e4, 64, 4096, 1, (0,)),
             ("const 1000", DEFAULT_TUNING[:2], "const", 0.5, 100, 1000, 1, (0,)),
             ("const 4096 strided", DEFAULT_TUNING[:2], "const", 0.5, 64, 4096, 32, (0, 6)))
    for name, (clen, halo), kind, lam, nf, ln, inc, ops in cases:
        lane_lib.proxtv_lane_tuning(clen, halo, -1)
        F = make(kind, nf, ln, rng)
        for op in ops:
            lane_lib.proxtv_lane_stats(1)
            check_op(emu, lane_lib, op, F, nf, ln, inc, lam, dt, rng, (name, op))
            reps = lane_lib.proxtv_lane_stats(1)
            assert reps > 0, (name, op)
            print("REPAIRS %s %s op %d: %d" % (np.dtype(dt).name, name, op, reps))


def test_refusals_leave_output_untouched(lane_lib):
    """Shapes the TMA tiling cannot take are refused before anything runs: return 0, proxtv_last_error() names the entry point, and
    the output buffer is untouched (callers fall back to the chunked engine)."""
    import torch
    dev = torch.device("cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for dt, fn, name in ((torch.float64, lane_lib.proxtv_lane_prox_dev_f64, "proxtv_lane_prox_dev_f64"),
                         (torch.float32, lane_lib.proxtv_lane_prox_dev_f32, "proxtv_lane_prox_dev_f32")):
        es = torch.tensor([], dtype=dt).element_size()
        buf = torch.randn(64 * 256 + 8, dtype=dt, device=dev)
        X = torch.full((64 * 256 + 8,), 7.0, dtype=dt, device=dev)
        cases = (("base off by one element", buf[1:], X, 64, 256, 1),
                 ("output off by one element", buf, X[1:], 64, 256, 1),
                 ("contig pitch not a multiple of 16 B", buf, X, 64, 16 // es + 1, 1),
                 ("strided pitch not a multiple of 16 B", buf, X, 2 * (16 // es + 1), 64, 16 // es + 1))
        for what, a, x, nf, ln, inc in cases:
            ok = fn(0, C.c_void_p(a.data_ptr()), None, None, C.c_void_p(x.data_ptr()), nf, ln, inc, 0.3, st)
            torch.cuda.synchronize()
            assert ok == 0, what
            assert lane_lib.proxtv_last_error().decode().startswith(name), (what, lane_lib.proxtv_last_error())
            assert bool((X == 7.0).all()), what
    # float32 has no two-result entry point; the single-result one refuses op 3 (it needs X2)
    a = torch.randn(64 * 64, dtype=torch.float32, device=dev); x = torch.full_like(a, 7.0)
    assert lane_lib.proxtv_lane_prox_dev_f32(3, C.c_void_p(a.data_ptr()), C.c_void_p(a.data_ptr()), C.c_void_p(a.data_ptr()),
                                             C.c_void_p(x.data_ptr()), 64, 64, 64, 0.3, st) == 0
    torch.cuda.synchronize()
    assert bool((x == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------- whole solves
def dyadic(shape, seed, dt):
    """cfg-2 style images (blocks + noise) on the grid integers / 256: exact in float32, and their sums exact in any order."""
    rng = np.random.default_rng(seed)
    B, M, N = shape
    Y = np.repeat(np.repeat(rng.normal(0, 1, (B, M // 8 + 1, N // 8 + 1)), 8, axis=1), 8, axis=2)[:, :M, :N] + rng.normal(0, 0.3, shape)
    return (np.round(Y * 256) / 256).astype(dt)


def dr_host(emu, Y, lam, maxit):
    """DR2_TV of every image of Y (B, M, N) with the lane engine's schedule (solver.cu: dr2_lane_body; dr2_lane_t_body computes the
    same expressions): t = 2 mean; per iteration x1 = prox_cols(t) (t itself in the first: the prox of a constant), d = t - x1,
    t' = d + prox_rows(Y - (2 d - t)); finally out = prox_rows(Y - d).  Arithmetic in the storage type; the start value is the
    float64 sum, doubled, divided by M N and rounded to the storage type (exact sums on dyadic inputs)."""
    T = Y.dtype.type
    B, M, N = Y.shape
    mean2 = (2.0 * Y.astype(np.float64).reshape(B, -1).sum(axis=1)) / float(M * N)
    t = np.ascontiguousarray(np.broadcast_to(mean2.astype(T)[:, None, None], Y.shape))
    lam = T(lam)

    def cols(a):
        return slope_fibers(emu, np.ascontiguousarray(a.transpose(0, 2, 1)), B * N, M, 1, lam).reshape(B, N, M).transpose(0, 2, 1)

    def rows(a):
        return slope_fibers(emu, np.ascontiguousarray(a), B * M, N, 1, lam).reshape(B, M, N)

    for it in range(maxit + 1):
        x1 = t.copy() if it == 0 else cols(t)
        d = t - x1
        if it == maxit:
            return rows(Y - d)
        t = d + rows(Y - (T(2) * d - t))


SHAPES = ((52, 36), (100, 140))       # M != N, multiples of 4 (the float32 pitch rule), not of 32
LAM = 0.375


@pytest.fixture(scope="module")
def host_solves(emu):
    cache = {}

    def get(shape, dt, maxit, batch=1, seed=0):
        key = (shape, np.dtype(dt).name, maxit, batch, seed)
        if key not in cache:
            cache[key] = dr_host(emu, dyadic((batch,) + shape, seed + 7 * batch, dt), LAM, maxit)
        return cache[key]
    return get


@pytest.mark.parametrize("maxit", [1, 2, 35])
@pytest.mark.parametrize("shape", SHAPES, ids=["52x36", "100x140"])
def test_dr2_lane_solves_bit_exact(ptv, engine, host_solves, shape, maxit):
    """Whole DR2_TV solves on both lane schedules, every entry path: numpy (column-major, staged or transposed schedule), torch
    row-major (transposed schedule, results written in place), torch column-major views, batches -- float64 and float32."""
    import torch
    M, N = shape
    it_arg = 0 if maxit == 35 else maxit                      # 0: the reference's default of 35 iterations
    for dt in (np.float64, np.float32):
        T = torch.float64 if dt == np.float64 else torch.float32
        Y1 = dyadic((1,) + shape, 7, dt); want1 = host_solves(shape, dt, maxit)
        Y3 = dyadic((3,) + shape, 21, dt); want3 = host_solves(shape, dt, maxit, batch=3)
        for eng in ("lane", "lane-t"):
            engine(eng)
            what = (shape, maxit, np.dtype(dt).name, eng)
            if dt == np.float64:
                got = ptv.tv1_2d(np.asfortranarray(Y1[0]), LAM, max_iters=it_arg)
                assert np.array_equal(got, want1[0]), what + ("numpy",)
            assert np.array_equal(ptv.tv1_2d_batched(Y1, LAM, max_iters=it_arg), want1), what + ("numpy batch 1",)
            assert np.array_equal(ptv.tv1_2d_batched(Y3, LAM, max_iters=it_arg), want3), what + ("numpy batch 3",)
            tr = torch.tensor(Y1[0], dtype=T, device="cuda")                               # row-major
            assert np.array_equal(ptv.tv1_2d(tr, LAM, max_iters=it_arg).cpu().numpy(), want1[0]), what + ("torch row-major",)
            tc = torch.tensor(np.ascontiguousarray(Y1[0].T), dtype=T, device="cuda").T     # column-major view
            oc = ptv.tv1_2d(tc, LAM, max_iters=it_arg)
            assert oc.stride() == tc.stride() and np.array_equal(oc.cpu().numpy(), want1[0]), what + ("torch column-major",)
            tb = torch.tensor(Y3, dtype=T, device="cuda")
            assert np.array_equal(ptv.tv1_2d_batched(tb, LAM, max_iters=it_arg).cpu().numpy(), want3), what + ("torch batch 3",)


def test_lane_schedules_agree_on_general_data(ptv, engine):
    """On general (not dyadic) column-major data the staged and the transposed schedules sum the start value over the same memory and
    execute the same expressions: bit-identical.  A row-major tensor sums it in another order: <= 1e-12 relative."""
    import torch
    Y = np.asfortranarray(O.gen_cfg2(100, 140, seed=3, block=8))
    res = {}
    for eng in ("lane", "lane-t"):
        engine(eng)
        res[eng] = (ptv.tv1_2d(Y, 0.2), ptv.tv1_2d_batched(np.stack([Y, 2 * Y]).astype(np.float32), 0.2))
        rm = ptv.tv1_2d(torch.tensor(np.ascontiguousarray(Y), device="cuda"), 0.2).cpu().numpy()
        assert relerr(rm, res[eng][0]) <= 1e-12, eng
    assert np.array_equal(res["lane"][0], res["lane-t"][0])
    assert np.array_equal(res["lane"][1], res["lane-t"][1])


def test_graph_replay_with_new_data(ptv, engine, host_solves, emu):
    """A solve is captured into a CUDA graph and replayed while the call's pointers stay the same: new data copied into the same
    tensors must give the host driver's result for the new data, call after call, in both storage orders and both dtypes."""
    import torch
    lib = ptv.load()
    M, N = SHAPES[1]
    engine("lane")
    for dt, fn in ((np.float64, lib.proxtv_DR2_TV_dev_f64), (np.float32, lib.proxtv_DR2_TV_dev_f32)):
        T = torch.float64 if dt == np.float64 else torch.float32
        Ya = dyadic((1, M, N), 7, dt); Yb = dyadic((1, M, N), 99, dt)
        wa = host_solves((M, N), dt, 2); wb = dr_host(emu, Yb, LAM, 2)
        for row_major in (1, 0):
            img = (lambda y: y[0]) if row_major else (lambda y: np.ascontiguousarray(y[0].T))    # column-major: the transpose, row-major
            Yt = torch.tensor(img(Ya), dtype=T, device="cuda"); out = torch.empty_like(Yt)
            info = np.zeros(3)
            st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            for k, (src, want) in enumerate(((Ya, wa), (Yb, wb), (Ya, wa), (Yb, wb))):
                Yt.copy_(torch.tensor(img(src), dtype=T))
                fn(M, N, 1, row_major, C.c_void_p(Yt.data_ptr()), LAM, LAM, C.c_void_p(out.data_ptr()), 2,
                   C.c_void_p(info.ctypes.data), st)
                assert info[2] != 3, lib.proxtv_last_error()
                got = out.cpu().numpy()
                got = got if row_major else got.T
                assert np.array_equal(got, want[0]), (np.dtype(dt).name, row_major, k)


def test_lane_fallback_edges(ptv, port, engine):
    """Shapes the lane engine refuses with the engine forced: the solve still runs (chunked engine) and matches the oracle."""
    import torch
    rng = np.random.default_rng(105)
    for eng in ("lane", "lane-t"):
        engine(eng)
        Y = rng.normal(size=(51, 40))
        tr = torch.tensor(Y, device="cuda")                                  # row-major with an odd dimension: pitch refused
        assert relerr(ptv.tv1_2d(tr, 0.3).cpu().numpy(), port.dr2_tv(Y, 0.3)[0]) <= 1e-9, eng
        Z = rng.normal(size=(48, 40))
        buf = torch.empty(48 * 40 + 1, dtype=torch.float64, device="cuda")
        tm = buf[1:].view(48, 40); tm.copy_(torch.tensor(Z))                 # storage offset of one element: misaligned base
        assert tm.storage_offset() == 1
        assert relerr(ptv.tv1_2d(tm, 0.3).cpu().numpy(), port.dr2_tv(Z, 0.3)[0]) <= 1e-9, eng
        for shape in ((1, 40), (40, 1)):
            V = np.asfortranarray(rng.normal(size=shape))
            assert relerr(ptv.tv1_2d(V, 0.3), port.dr2_tv(V, 0.3)[0]) <= 1e-9, (eng, shape)


# A fresh process: the lane engine's scratch is grow-only and process-wide, so only a process that starts with none controls which
# call makes it grow.
_GROWTH = r"""
import ctypes as C, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import proxtv_b200 as ptv
lib = ptv.require_device()
ptv.set_engine("lane"); lib.proxtv_lane_tuning(0, 32, -1)
d = np.load(sys.argv[2])
Y = torch.tensor(np.ascontiguousarray(d["Y"].T), device="cuda")     # column-major image
big = torch.tensor(d["big"], device="cuda")
nf, ln, lam = int(d["nf"]), int(d["ln"]), float(d["lam"])
M, N = d["Y"].shape
out = torch.empty_like(Y); xb = torch.empty_like(big); info = np.zeros(3)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
res = {}
for k in range(2):
    lib.proxtv_DR2_TV_dev_f64(M, N, 1, 0, C.c_void_p(Y.data_ptr()), 0.375, 0.375, C.c_void_p(out.data_ptr()), 3, C.c_void_p(info.ctypes.data), st)
    res["a%d" % k] = out.t().cpu().numpy()
    xb.fill_(float("nan"))
    ok = lib.proxtv_lane_prox_dev_f64(0, C.c_void_p(big.data_ptr()), None, None, C.c_void_p(xb.data_ptr()), nf, ln, nf, lam, st)
    assert ok == 1, lib.proxtv_last_error()
    res["big%d" % k] = xb.cpu().numpy().ravel()
np.savez(sys.argv[3], **res)
"""


def test_graph_survives_lane_scratch_growth(emu, tmp_path):
    """Solve A (captured into a graph) -> a lane call with many more fibers (the scratch grows: freed and allocated again, possibly at
    the same address, with a larger counter region) -> solve A again -> the large call again, lambda large enough that every fiber
    needs the verification and repair steered by the group counters.  A replayed graph that kept the old layout would write its chunk
    records into what are now counters; every result must still be the host reference's, whichever address the allocator returned."""
    Y = dyadic((1, 64, 48), 5, np.float64)
    nf, ln, lam = 8192, 300, 1e4
    big = np.ascontiguousarray(make("blocks", nf, ln, np.random.default_rng(106)).T)     # (ln, nf): strided fibers, inc = nf
    src = tmp_path / "in.npz"; dst = tmp_path / "out.npz"
    np.savez(src, Y=Y[0], big=big, nf=nf, ln=ln, lam=lam)
    r = subprocess.run([sys.executable, "-c", _GROWTH, ROOT, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(dst)
    wa = dr_host(emu, Y, LAM, 3)[0]
    wb = slope_fibers(emu, big.ravel(), nf, ln, nf, lam)
    for k in range(2):
        assert np.array_equal(got["a%d" % k], wa), k
        assert np.array_equal(got["big%d" % k], wb), ("large call", k, first_diff(got["big%d" % k], wb, nf, ln, nf, False))
