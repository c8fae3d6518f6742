"""The numpy front end against a recording fake of the library: for every public function, dtype, memory order, single and batched
form, method, iteration cap and empty input, the C calls it makes (symbol, scalar arguments, which pointers are NULL), the result's
dtype, shape and order, which calls raise when the entry point returns 0 or writes RC = 3 into an info row, and which
``last_info`` the call sets.  The fake copies each entry point's input array to its output, so a result equal to the input also
shows that the front end reads the output in the layout it wrote the input in."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import proxtv_b200 as ptv
from proxtv_b200 import _lib

P = "P"                   # a non-NULL pointer argument in an expected call
RC_ERROR = 3


def _prod(a, i, k):
    return int(np.prod(np.ctypeslib.as_array((C.c_int * int(a[k])).from_address(a[i])), dtype=np.int64))


# The host entry points the numpy paths call (include/proxtv_b200.h): the position of `info` (None: no info), the argument holding
# the number of info rows (None: one), the input and output arrays, and their element count.
_HOST = {
    "proxtv_prox_fibers": (None, None, 0, 1, lambda a: a[2] * a[3]),
    "DR2_TV": (10, None, 2, 7, lambda a: a[0] * a[1]),
    "DR2L1W_TV": (8, None, 2, 5, lambda a: a[0] * a[1]),
    "CondatChambollePock2_TV": (7, None, 2, 4, lambda a: a[0] * a[1]),
    "PD2_TV": (5, None, 0, 4, lambda a: _prod(a, 6, 7)),
    "PD_TV": (5, None, 0, 4, lambda a: _prod(a, 6, 7)),
    "PDR_TV": (5, None, 0, 4, lambda a: _prod(a, 6, 7)),
    "proxtv_PD_TV": (4, None, 0, 3, lambda a: _prod(a, 5, 6)),                       # proxtv_PD_TV_f32
    "proxtv_DR2_TV_batched": (8, None, 3, 6, lambda a: a[0] * a[1] * a[2]),
    "proxtv_DR2L1W_TV_batched": (9, None, 4, 7, lambda a: a[0] * a[1] * a[2]),
    "proxtv_CP2_TV_batched": (9, 2, 4, 6, lambda a: a[0] * a[1] * a[2]),
    "proxtv_CP2W_TV_batched": (10, 2, 4, 7, lambda a: a[0] * a[1] * a[2]),
    "proxtv_PD_TV_batched": (4, 8, 0, 3, lambda a: _prod(a, 5, 6) * a[8]),
    "proxtv_PD2_TV_batched": (4, 8, 0, 3, lambda a: _prod(a, 5, 6) * a[8]),
}

# The reference-named single-image symbols run the same body, with the same arguments, as the batched host symbol with batch = 1
# (proxtv_b200/csrc/capi.cu, Part 1 and the _batched_ thunks), so both spellings of a call map to one key.
_SAME_AS_BATCHED = {
    # DR2_TV(M, N, Y, W1, W2, 1, 1, out, n_threads, maxit, info) -> run_dr2(host_io, M, N, 1, 0, ...) = proxtv_DR2_TV_batched_f64
    "DR2_TV": lambda a: ("proxtv_DR2_TV_batched_f64", [a[0], a[1], 1, a[2], a[3], a[4], a[7], a[9], a[10]]),
    # DR2L1W_TV(M, N, Y, W1, W2, out, n_threads, maxit, info) -> run_drw(host_io, M, N, 1, 0, ...) = proxtv_DR2L1W_TV_batched_f64
    "DR2L1W_TV": lambda a: ("proxtv_DR2L1W_TV_batched_f64", [a[0], a[1], 1, 0, a[2], a[3], a[4], a[5], a[7], a[8]]),
    # CondatChambollePock2_TV(M, N, Y, lambda, X, alg, maxit, info) -> run_cp2(host_io, M, N, 1, 0, ...) = proxtv_CP2_TV_batched_f64
    "CondatChambollePock2_TV": lambda a: ("proxtv_CP2_TV_batched_f64", [a[0], a[1], 1, 0, a[2], a[3], a[4], a[5], a[6], a[7]]),
}


def _spec(name):
    base = name[:-4] if name.endswith(("_f32", "_f64")) else name
    return _HOST[base]


def _raw(a):
    if isinstance(a, C.c_void_p):
        return a.value
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a


def canon(name, args):
    """(symbol, arguments) with every pointer as P or None, the reference-named symbols as their batched key."""
    if name == "DR2_TV":
        assert args[5] == 1.0 and args[6] == 1.0
    if name in _SAME_AS_BATCHED:
        name, args = _SAME_AS_BATCHED[name](args)
    types = _lib.SIGNATURES[name][1]
    return (name,) + tuple((None if v is None else P) if t is C.c_void_p else v for v, t in zip(args, types))


class FakeLib:
    """Stands in for the ctypes handle: one device, every call recorded.  mode 'ok': copy the input to the output, fill each info row
    with [7 + row, 0.5, 0] and return 1; 'zero': return 0 and write nothing; 'rc3': as 'ok', with RC = 3 in the last info row."""

    def __init__(self):
        self.calls, self.mode, self.infos, self.pooled = [], "ok", [], []

    def proxtv_device_count(self):
        return 1

    def proxtv_last_error(self):
        return b"fake: refused"

    def __getattr__(self, name):
        if name not in _lib.SIGNATURES:
            raise AttributeError(name)

        def call(*args):
            a = [_raw(v) for v in args]
            assert len(a) == len(_lib.SIGNATURES[name][1]), name
            self.calls.append((name, a))
            if self.mode == "zero":
                return 0
            info_at, rows_at, i, o, count = _spec(name)
            n = int(count(a))
            if n:
                C.memmove(a[o], a[i], n * (4 if name.endswith("_f32") else 8))
            if info_at is not None and a[info_at]:
                rows = max(int(a[rows_at]), 1) if rows_at is not None else 1
                info = np.ctypeslib.as_array((C.c_double * (3 * rows)).from_address(a[info_at])).reshape(rows, 3)
                info[:] = [[7 + r, 0.5, 0] for r in range(rows)]
                if self.mode == "rc3":
                    info[-1, 2] = RC_ERROR
                self.infos.append(info.copy())
            return 1
        return call


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "_lib", lib)
    prev = ptv.set_pinned_results(False)
    empty = ptv._pool.empty
    monkeypatch.setattr(ptv._pool, "empty", lambda *a: lib.pooled.append(a) or empty(*a))
    yield lib
    ptv.set_pinned_results(prev)


# ---- the cases --------------------------------------------------------------------------------------------------------------------
# (id, call, expected calls, result dtype, shape, order ("C", "F", "CF" both, "" neither), whether a zero return raises, the function
#  whose last_info the call sets, the result's values).  The 2D functions, tvgen and tvgen_pdr take their result from the pinned pool.
_OWNERS = (ptv.tvgen, ptv.tvgen_pdr, ptv.tvgen_batched)
_CP = {"condat": 0, "chambolle-pock": 1, "chambolle-pock-acc": 2}
W = 0.25


def _x(shape, dt, order, seed=0):
    return np.asarray(np.random.default_rng(seed).normal(size=shape), dtype=dt, order=order)


def _flags(a):
    return ("C" if a.flags.c_contiguous else "") + ("F" if a.flags.f_contiguous else "")


def _cases():
    out = []

    def add(id_, fn, calls, dt, shape, order, rc, owner=None, value=None):
        pooled = "1d" not in id_ and "tvgen_batched" not in id_
        out.append(pytest.param(fn, calls, np.dtype(dt), tuple(shape), order, rc, owner, value, pooled, id=id_))

    for dt in (np.float64, np.float32):
        s = np.dtype(dt).name[-2:]
        sfx = "_f32" if dt == np.float32 else "_f64"
        for o in ("C", "F"):
            # ---- 1D ----
            x = _x((3, 4), dt, o)
            add("tv1_1d-%s-%s" % (s, o), lambda x=x: ptv.tv1_1d(x, W),
                [("proxtv_prox_fibers_f64", P, P, 1, 12, 1, W, None)], np.float64, (12,), "CF", True,
                value=x.ravel(order=o).astype(np.float64))
            x1 = _x(7, dt, o)
            w1 = np.abs(_x(6, np.float64, o, 1))
            add("tv1w_1d-%s-%s" % (s, o), lambda x=x1, w=w1: ptv.tv1w_1d(x, w),
                [("proxtv_prox_fibers_f64", P, P, 1, 7, 1, 0.0, P)], np.float64, (7,), "CF", True, value=x1.astype(np.float64))
            xb = _x((3, 9), dt, o)
            add("tv1_1d_batched-%s-%s" % (s, o), lambda x=xb: ptv.tv1_1d_batched(x, W),
                [("proxtv_prox_fibers" + sfx, P, P, 3, 9, 1, W, None)], dt, (3, 9), "C", True)
            wb = np.abs(_x((3, 8), np.float64, o, 1))
            add("tv1w_1d_batched-%s-%s" % (s, o), lambda x=xb, w=wb: ptv.tv1w_1d_batched(x, w),
                [("proxtv_prox_fibers" + sfx, P, P, 3, 9, 1, 0.0, P)], dt, (3, 9), "C", True)
            # ---- 2D, single image ----
            x2 = _x((5, 4), dt, o)
            wc, wr = np.abs(_x((4, 4), np.float64, o, 1)), np.abs(_x((5, 3), np.float64, o, 2))
            for mi in (0, 3):
                add("tv1_2d-dr-%s-%s-%d" % (s, o, mi), lambda x=x2, mi=mi: ptv.tv1_2d(x, W, max_iters=mi),
                    [("proxtv_DR2_TV_batched_f64", 5, 4, 1, P, W, W, P, mi, P)], np.float64, (5, 4), "F", False,
                    value=x2.astype(np.float64))
                add("tv1_2d-pd-%s-%s-%d" % (s, o, mi), lambda x=x2, mi=mi: ptv.tv1_2d(x, W, max_iters=mi, method="pd"),
                    [("PD2_TV", P, P, P, P, P, P, P, 2, 2, 1, mi)], np.float64, (5, 4), "F", True, value=x2.astype(np.float64))
                for m, alg in _CP.items():
                    add("tv1_2d-%s-%s-%s-%d" % (m, s, o, mi), lambda x=x2, mi=mi, m=m: ptv.tv1_2d(x, W, max_iters=mi, method=m),
                        [("proxtv_CP2_TV_batched_f64", 5, 4, 1, 0, P, W, P, alg, mi, P)], np.float64, (5, 4), "F", True,
                        value=x2.astype(np.float64))
                add("tv1w_2d-dr-%s-%s-%d" % (s, o, mi), lambda x=x2, mi=mi: ptv.tv1w_2d(x, wc, wr, max_iters=mi),
                    [("proxtv_DR2L1W_TV_batched_f64", 5, 4, 1, 0, P, P, P, P, mi, P)], np.float64, (5, 4), "F", False,
                    value=x2.astype(np.float64))
                for m in ("condat", "chambolle-pock"):
                    add("tv1w_2d-%s-%s-%s-%d" % (m, s, o, mi), lambda x=x2, mi=mi, m=m: ptv.tv1w_2d(x, wc, wr, max_iters=mi, method=m),
                        [("proxtv_CP2W_TV_batched_f64", 5, 4, 1, 0, P, P, P, P, _CP[m], mi, P)], np.float64, (5, 4), "F", True,
                        value=x2.astype(np.float64))
            # ---- 2D, batched ----
            x3 = _x((3, 5, 4), dt, o)
            wc3, wr3 = np.abs(_x((3, 4, 4), np.float64, o, 1)), np.abs(_x((3, 5, 3), np.float64, o, 2))
            for mi in (0, 3):
                add("tv1_2d_batched-dr-%s-%s-%d" % (s, o, mi), lambda x=x3, mi=mi: ptv.tv1_2d_batched(x, W, max_iters=mi),
                    [("proxtv_DR2_TV_batched" + sfx, 5, 4, 3, P, W, W, P, mi, P)], dt, (3, 5, 4), "", False)
                for m, alg in _CP.items():
                    add("tv1_2d_batched-%s-%s-%s-%d" % (m, s, o, mi), lambda x=x3, mi=mi, m=m: ptv.tv1_2d_batched(x, W, max_iters=mi, method=m),
                        [("proxtv_CP2_TV_batched" + sfx, 5, 4, 3, 1, P, W, P, alg, mi, P)], dt, (3, 5, 4), "C", True)
                add("tv1w_2d_batched-dr-%s-%s-%d" % (s, o, mi), lambda x=x3, mi=mi: ptv.tv1w_2d_batched(x, wc3, wr3, max_iters=mi),
                    [("proxtv_DR2L1W_TV_batched" + sfx, 5, 4, 3, 1, P, P, P, P, mi, P)], dt, (3, 5, 4), "C", False)
                for m in ("condat", "chambolle-pock"):
                    add("tv1w_2d_batched-%s-%s-%s-%d" % (m, s, o, mi),
                        lambda x=x3, mi=mi, m=m: ptv.tv1w_2d_batched(x, wc3, wr3, max_iters=mi, method=m),
                        [("proxtv_CP2W_TV_batched" + sfx, 5, 4, 3, 1, P, P, P, P, _CP[m], mi, P)], dt, (3, 5, 4), "C", True)
            # ---- N-D ----
            xn = _x((4, 3, 5), dt, o)
            for mi in (0, 3):
                for k, ds in ((3, [1, 2, 3]), (2, [1, 3]), (1, [2])):
                    ws = [0.1, 0.2, 0.3][:k]
                    if k == 2:
                        sym, odt = ("PD2_TV", P, P, P, P, P, P, P, 3, 2, 1, mi), np.float64
                    elif dt == np.float32:
                        sym, odt = ("proxtv_PD_TV_f32", P, P, P, P, P, P, 3, k, mi), np.float32
                    else:
                        sym, odt = ("PD_TV", P, P, P, P, P, P, P, 3, k, 1, mi), np.float64
                    add("tvgen-%d-%s-%s-%d" % (k, s, o, mi), lambda x=xn, ws=ws, ds=ds, mi=mi: ptv.tvgen(x, ws, ds, [1] * len(ws), max_iters=mi),
                        [sym], odt, (4, 3, 5), "F", True, ptv.tvgen, value=xn.astype(odt))
                    db = [d for d in ds if d < 3]                                       # axes of an item of shape (3, 5)
                    bsym = "proxtv_%s_batched%s" % ("PD2_TV" if len(db) == 2 else "PD_TV", sfx)
                    add("tvgen_batched-%d-%s-%s-%d" % (len(db), s, o, mi),
                        lambda x=xn, db=db, mi=mi: ptv.tvgen_batched(x, [0.1, 0.2][:len(db)], db, [1] * len(db), max_iters=mi),
                        [(bsym, P, P, P, P, P, P, 2, len(db), 4, mi)], dt, (4, 3, 5), "", True, ptv.tvgen_batched)
                add("tvgen_pdr-%s-%s-%d" % (s, o, mi), lambda x=xn, mi=mi: ptv.tvgen_pdr(x, [0.1, 0.2], [1, 3], [1, 1], max_iters=mi),
                    [("PDR_TV", P, P, P, P, P, P, P, 3, 2, 1, mi)], np.float64, (4, 3, 5), "F", True, ptv.tvgen_pdr,
                    value=xn.astype(np.float64))
        # ---- empty inputs ----
        add("empty-tv1_1d-%s" % s, lambda dt=dt: ptv.tv1_1d(np.zeros((0, 3), dt), W), [], np.float64, (0,), "CF", True)
        add("single-tv1w_1d-%s" % s, lambda dt=dt: ptv.tv1w_1d(np.full(1, 2.5, dt), np.zeros(0)), [], np.float64, (1,), "CF", True)
        add("empty-tv1_1d_batched-%s" % s, lambda dt=dt: ptv.tv1_1d_batched(np.zeros((0, 5), dt), W), [], dt, (0, 5), "CF", True)
        add("empty-tv1w_1d_batched-%s" % s, lambda dt=dt: ptv.tv1w_1d_batched(np.zeros((0, 5), dt), np.zeros((0, 4))), [], dt, (0, 5), "CF", True)
        add("empty-tv1_2d-dr-%s" % s, lambda dt=dt: ptv.tv1_2d(np.zeros((0, 5), dt), W),
            [("proxtv_DR2_TV_batched_f64", 0, 5, 1, P, W, W, P, 0, P)], np.float64, (0, 5), "CF", False)
        add("empty-tv1_2d-pd-%s" % s, lambda dt=dt: ptv.tv1_2d(np.zeros((0, 5), dt), W, method="pd"),
            [("PD2_TV", P, P, P, P, P, P, P, 2, 2, 1, 0)], np.float64, (0, 5), "CF", True)
        add("empty-tv1_2d-condat-%s" % s, lambda dt=dt: ptv.tv1_2d(np.zeros((0, 5), dt), W, method="condat"),
            [("proxtv_CP2_TV_batched_f64", 0, 5, 1, 0, P, W, P, 0, 0, P)], np.float64, (0, 5), "CF", True)
        for shp in ((0, 5, 4), (2, 0, 4)):
            e = "x".join(map(str, shp))
            sfx = "_f32" if dt == np.float32 else "_f64"
            add("empty-tv1_2d_batched-dr-%s-%s" % (e, s), lambda shp=shp, dt=dt: ptv.tv1_2d_batched(np.zeros(shp, dt), W),
                [("proxtv_DR2_TV_batched" + sfx, shp[1], shp[2], shp[0], P, W, W, P, 0, P)], dt, shp, "", False)
            add("empty-tv1_2d_batched-condat-%s-%s" % (e, s), lambda shp=shp, dt=dt: ptv.tv1_2d_batched(np.zeros(shp, dt), W, method="condat"),
                [], dt, shp, "CF", True)
        for m in ("dr", "condat"):
            add("empty-tv1w_2d_batched-%s-%s" % (m, s),
                lambda m=m, dt=dt: ptv.tv1w_2d_batched(np.zeros((0, 5, 4), dt), np.zeros((0, 4, 4)), np.zeros((0, 5, 3)), method=m),
                [], dt, (0, 5, 4), "CF", True)
        add("empty-tvgen-%s" % s, lambda dt=dt: ptv.tvgen(np.zeros((0, 3), dt), [0.1], [1], [1]),
            [("proxtv_PD_TV_f32", P, P, P, P, P, P, 2, 1, 0) if dt == np.float32 else ("PD_TV", P, P, P, P, P, P, P, 2, 1, 1, 0)],
            dt, (0, 3), "CF", True, ptv.tvgen)
        add("empty-tvgen_pdr-%s" % s, lambda dt=dt: ptv.tvgen_pdr(np.zeros((0, 3), dt), [0.1], [1], [1]),
            [("PDR_TV", P, P, P, P, P, P, P, 2, 1, 1, 0)], np.float64, (0, 3), "CF", True, ptv.tvgen_pdr)
        add("empty-tvgen_batched-B0-%s" % s, lambda dt=dt: ptv.tvgen_batched(np.zeros((0, 3, 2), dt), [0.1], [1], [1]),
            [], dt, (0, 3, 2), "CF", True, ptv.tvgen_batched)
        add("empty-tvgen_batched-item-%s" % s, lambda dt=dt: ptv.tvgen_batched(np.zeros((2, 0, 3), dt), [0.1], [1], [1]),
            [("proxtv_PD_TV_batched" + ("_f32" if dt == np.float32 else "_f64"), P, P, P, P, P, P, 2, 1, 2, 0)],
            dt, (2, 0, 3), "CF", True, ptv.tvgen_batched)
    return out


def _set_sentinels():
    for f in _OWNERS:
        f.last_info = "unset"


def _owner(owner):
    changed = [f for f in _OWNERS if not (isinstance(f.last_info, str) and f.last_info == "unset")]
    assert changed == ([owner] if owner is not None else []), [f.__name__ for f in changed]


@pytest.mark.parametrize("fn, calls, dt, shape, order, rc, owner, value, pooled", _cases())
def test_numpy_front_end(fake, fn, calls, dt, shape, order, rc, owner, value, pooled):
    _set_sentinels()
    y = fn()
    assert [canon(n, a) for n, a in fake.calls] == [tuple(c) for c in calls]
    assert isinstance(y, np.ndarray) and y.dtype == dt and y.shape == shape
    assert _flags(y) == order if y.size > 1 else True
    if value is not None:
        assert np.array_equal(y, value)
    assert [(tuple(s), np.dtype(d)) for s, d, _ in fake.pooled] == ([(y.shape if order else y.shape[:1] + y.shape[:0:-1], dt)] if pooled else [])
    _owner(owner)
    if owner is not None:
        rows = [i for i in fake.infos]
        want = rows[-1] if rows else np.zeros((0, 3))
        got = owner.last_info
        if owner is ptv.tvgen_batched:
            assert got.shape == (shape[0], 3) and np.array_equal(got, want)
        else:
            assert got.shape == (3,) and np.array_equal(got, want[0])
    # a zero return, then RC = 3 in the last info row
    for mode, raises in (("zero", rc and bool(calls)), ("rc3", any(_spec(n)[0] is not None for n, _ in fake.calls))):
        fake.calls, fake.infos, fake.mode = [], [], mode
        _set_sentinels()
        if raises:
            with pytest.raises(ptv.ProxTVError):
                fn()
            _owner(None)
        else:
            fn()
            _owner(owner)
        assert [canon(n, a) for n, a in fake.calls] == [tuple(c) for c in calls]
        fake.mode = "ok"


def test_single_image_values_reach_the_right_arguments(fake):
    """Scalars that the generic expectations above cannot tell apart: the ignored n_threads of the DR entry points, and PD2_TV's
    norms and dims of tv1_2d(method='pd')."""
    x = _x((5, 4), np.float64, "F")
    ptv.tv1_2d(x, W, n_threads=4, method="pd")
    (_, a), = fake.calls
    assert a[9] == 4
    for i, want in ((1, [W, W]), (2, [1.0, 1.0]), (3, [1.0, 2.0])):
        assert np.array_equal(np.ctypeslib.as_array((C.c_double * 2).from_address(a[i])), want)


def test_tvgen_hands_a_float64_ws_to_the_solver_itself(fake):
    """PD_TV / PDR_TV scale their lambdas in place, so the numpy tvgen / tvgen_pdr pass a float64 ndarray ws itself (the reference's
    quirk); tvgen_batched passes a copy."""
    x = _x((4, 3, 5), np.float64, "F")
    for f in (ptv.tvgen, ptv.tvgen_pdr):
        ws = np.array([0.1, 0.2, 0.3])
        fake.calls = []
        f(x, ws, [1, 2, 3], [1, 1, 1])
        assert fake.calls[0][1][1] == ws.ctypes.data
    ws = np.array([0.1, 0.2, 0.3])
    fake.calls = []
    ptv.tvgen_batched(x, ws, [1, 2, 1], [1, 1, 1])
    assert fake.calls[0][1][1] != ws.ctypes.data


def test_errors_before_the_library(fake):
    """Bad input raises its own exception type without a library call."""
    x2, x3 = np.zeros((5, 4)), np.zeros((2, 5, 4))
    for f, exc in ((lambda: ptv.tv1_2d(x2, -1.0), AssertionError),
                   (lambda: ptv.tv1_2d(x2, W, method="yang"), NotImplementedError),
                   (lambda: ptv.tv1_2d(x3, W), AssertionError),
                   (lambda: ptv.tv1_2d(x3, W, method="condat"), AssertionError),
                   (lambda: ptv.tv1_2d_batched(x2, W), AssertionError),
                   (lambda: ptv.tv1_2d_batched(x2, W, method="condat"), AssertionError),
                   (lambda: ptv.tv1_2d_batched(x3, W, method="pd"), AssertionError),
                   (lambda: ptv.tv1w_2d(x2, np.ones((4, 4)), np.ones((5, 4))), AssertionError),
                   (lambda: ptv.tv1w_2d(x2, -np.ones((4, 4)), np.ones((5, 3)), method="condat"), AssertionError),
                   (lambda: ptv.tvgen(x3, [0.1], [1], [2]), NotImplementedError),
                   (lambda: ptv.tvgen(x3, [0.1], [1, 2], [1]), AssertionError),
                   (lambda: ptv.tvgen_pdr(x3, [0.1], [1], [2]), NotImplementedError),
                   (lambda: ptv.tvgen_pdr(x3, [0.1], [1], [1], n_threads=0), AssertionError),
                   (lambda: ptv.tvgen_batched(x3, [0.1], [1], [2]), NotImplementedError),
                   (lambda: ptv.tvgen_batched(x3[0, 0], [0.1], [1], [1]), AssertionError),
                   (lambda: ptv.tv1_1d_batched(x3, W), AssertionError),
                   (lambda: ptv.tv1w_1d_batched(x2, np.ones((5, 4))), AssertionError)):
        with pytest.raises(exc):
            f()
    assert fake.calls == []


def test_numpy_calls_leave_torch_unimported():
    code = ("import sys; sys.path.insert(0, %r); import test_frontend_cpu as T, proxtv_b200 as ptv\n"
            "lib = T.FakeLib(); T._lib._lib = lib; ptv.set_pinned_results(False)\n"
            "for p in T._cases():\n"
            "    p.values[0]()\n"
            "assert len(lib.calls) > 50\n"
            "assert 'torch' not in sys.modules, 'torch imported'\n" % os.path.dirname(os.path.abspath(__file__)))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
