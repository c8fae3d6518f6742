"""The C ABI's refusals, entry point by entry point: the return value, proxtv_last_error(), the "<fn>: <msg>" line on stdout,
which info slots are written, and that outputs, tapes and lambdas are left alone.

Argument refusals that come before any device work run everywhere; the no-device refusals run only where no CUDA device is
present (like test_abi.py::test_fails_loudly_without_device), and a few refusals only a device can reach are marked gpu."""
import numpy as np
import pytest

import proxtv_b200
from proxtv_b200 import _lib

NODEV = "no usable CUDA device (libproxtv_b200 has no CPU fallback)"
INFO0 = 0.5                                            # what every info slot holds before the call
HAS_DEVICE = proxtv_b200.load().proxtv_device_count() != 0


class Bufs:
    def __init__(self):
        rng = np.random.default_rng(0)
        self.y = rng.normal(size=256)
        self.w = rng.uniform(0.1, 0.2, size=256)
        self.out, self.out2, self.out3 = (np.full(256, -7.0) for _ in range(3))
        self.tape = np.full(1 << 16, 0xAB, np.uint8)
        self.F = np.full(64, 0xDEADBEEF, np.uint32)
        self.U = np.full(64, 0xDEADBEEF, np.uint32)
        self.info = np.full(12, INFO0)
        self.lam = np.array([0.1, 0.2])
        self.neg = np.array([-0.1, 0.2])
        self.dims = np.array([1.0, 2.0])
        self.baddims = np.array([1.0, 5.0])
        self.ns = np.array([4, 4], np.int32)
        self.nsneg = np.array([4, -1], np.int32)

    def __getattr__(self, name):                       # b.p_<buf>: the buffer's address
        if name.startswith("p_"):
            return getattr(self, name[2:]).ctypes.data
        raise AttributeError(name)


def _canary(lib):
    """Leaves a known message in proxtv_last_error(), so that a refusal that writes none can be told apart."""
    assert lib.proxtv_prox_fibers_vjp_dev_f64(None, None, None, None, -1, 0, 1, 0.1, None, None) == 0
    return _lib.last_error()


def _check(capfd, sym, args, rc, msg, info=None, fn=None):
    """Calls sym(*args(b)); msg None: no message (the canary stays, nothing on stdout); info: {slot: value}, every other slot unchanged."""
    lib = proxtv_b200.load()
    b = Bufs()
    canary = _canary(lib)
    capfd.readouterr()
    keep = {k: getattr(b, k).copy() for k in ("y", "w", "out", "out2", "out3", "tape", "F", "U", "lam", "neg", "dims", "baddims", "ns")}
    got = getattr(lib, sym)(*args(b))
    out = capfd.readouterr().out
    assert got == rc, (sym, got)
    if msg is None:
        assert _lib.last_error() == canary and out == "", (sym, _lib.last_error(), out)
    else:
        line = "%s: %s" % (fn or sym, msg)
        assert _lib.last_error() == line and out == line + "\n", (sym, _lib.last_error(), out)
    want = np.full(12, INFO0)
    for k, v in (info or {}).items():
        want[k] = v
    assert np.array_equal(b.info, want), (sym, b.info)
    for k, v in keep.items():
        assert np.array_equal(getattr(b, k), v), (sym, k)


ALL3 = {2: 3, 5: 3, 8: 3}                              # info[3 b + RC] = RC_ERROR for the 3 items of a batch
ROW0 = {2: 3}


# (symbol, args(b), return, message or None, info slots written, name in the message when it is not the symbol)
ARG_CASES = []
NODEV_CASES = []


def _add(lst, sym, args, rc, msg, info=None, fn=None):
    lst.append(pytest.param(sym, args, rc, msg, info, fn, id="%s-%d" % (sym, sum(1 for p in lst if p.values[0] == sym))))


for t in ("f64", "f32"):
    # batched 1D prox, host arrays
    s = "proxtv_prox_fibers_" + t
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_out, 0, 8, 1, 0.1, None), 1, None)
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_out, 4, 8, 0, 0.1, None), 0, "invalid fiber geometry (need inc >= 1 and nf a multiple of inc)")
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_out, 4, 8, 3, 0.1, None), 0, "invalid fiber geometry (need inc >= 1 and nf a multiple of inc)")
    _add(NODEV_CASES, s, lambda b: (b.p_y, b.p_out, 4, 8, 1, 0.1, None), 0, NODEV)
    _add(NODEV_CASES, s, lambda b: (b.p_y, b.p_out, 4, 8, 1, 0.0, b.p_w), 0, NODEV)
    # batched 1D prox, device arrays
    _add(NODEV_CASES, "proxtv_prox_fibers_dev_" + t, lambda b: (b.p_y, b.p_out, 4, 8, 1, 0.1, None, None), 0, NODEV)
    # its backward
    s = "proxtv_prox_fibers_vjp_dev_" + t
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_y, b.p_out, None, 4, 8, 0, 0.1, None, None), 0,
         "invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1)")
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_y, b.p_out, None, 0, 8, 1, 0.1, None, None), 1, None)
    _add(ARG_CASES, s, lambda b: (b.p_y, None, b.p_out, None, 4, 8, 1, 0.1, None, None), 0, "NULL array")
    _add(ARG_CASES, s, lambda b: (b.p_y, b.p_y, b.p_out, None, 4, 8, 1, -0.1, None, None), 0, "negative penalty")
    _add(NODEV_CASES, s, lambda b: (b.p_y, b.p_y, b.p_out, b.p_out2, 4, 8, 1, 0.0, b.p_w, None), 0, NODEV)
    # segmentation tape of the 1D prox and the backward from it
    s = "proxtv_fiber_tape_dev_" + t
    geo = "invalid fiber geometry (need nf >= 0, len >= 0, inc >= 1, nf a multiple of inc)"
    _add(ARG_CASES, s, lambda b: (b.p_y, 4, 8, 3, 0.1, None, b.p_F, b.p_U, None), 0, geo)
    _add(ARG_CASES, s, lambda b: (b.p_y, 0, 8, 1, 0.1, None, b.p_F, b.p_U, None), 1, None)
    _add(ARG_CASES, s, lambda b: (b.p_y, 4, 8, 1, 0.1, None, None, b.p_U, None), 0, "NULL array")
    _add(ARG_CASES, s, lambda b: (b.p_y, 4, 8, 1, -0.1, None, b.p_F, b.p_U, None), 0, "negative penalty")
    _add(NODEV_CASES, s, lambda b: (b.p_y, 4, 8, 1, 0.1, None, b.p_F, b.p_U, None), 0, NODEV)
    s = "proxtv_prox_fibers_vjp_tape_dev_" + t
    _add(ARG_CASES, s, lambda b: (b.p_F, b.p_U, b.p_y, b.p_out, None, -1, 8, 1, None), 0, geo)
    _add(ARG_CASES, s, lambda b: (b.p_F, b.p_U, b.p_y, b.p_out, None, 4, 0, 1, None), 1, None)
    _add(ARG_CASES, s, lambda b: (b.p_F, b.p_U, None, b.p_out, None, 4, 8, 1, None), 0, "NULL array")
    _add(NODEV_CASES, s, lambda b: (b.p_F, b.p_U, b.p_y, b.p_out, None, 4, 8, 1, None), 0, NODEV)

    # DR2_TV: the solve (device and host arrays), the recorded solve, the backward
    _add(NODEV_CASES, "proxtv_DR2_TV_dev_" + t, lambda b: (4, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_info, None), 0, NODEV, ROW0)
    _add(NODEV_CASES, "proxtv_DR2_TV_batched_" + t, lambda b: (4, 4, 3, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_info), 0, NODEV, ROW0)
    _add(NODEV_CASES, "proxtv_DR2_TV_batched_" + t, lambda b: (4, 4, -1, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_info), 0, NODEV, ROW0)
    s = "proxtv_DR2_TV_record_dev_" + t
    _add(ARG_CASES, s, lambda b: (0, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0,
         "invalid shape (need M, N, batch >= 1)", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, None, 1 << 16, b.p_info, None), 0, "NULL array", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, 1, 0, b.p_y, 0.1, -0.1, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, "negative penalty", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_tape, 16, b.p_info, None), 0,
         "tape_bytes smaller than proxtv_DR2_TV_tape_bytes()", ROW0)
    _add(NODEV_CASES, s, lambda b: (4, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, NODEV, ROW0)
    _add(NODEV_CASES, s, lambda b: (4, 4, 1, 0, b.p_y, 0.1, 0.1, b.p_out, 5, b.p_tape, 1 << 16, None, None), 0, NODEV)
    s = "proxtv_DR2_TV_vjp_dev_" + t
    _add(ARG_CASES, s, lambda b: (4, 4, 0, 0, 5, b.p_tape, b.p_y, b.p_out, None, None), 0, "invalid shape (need M, N, batch >= 1)")
    _add(ARG_CASES, s, lambda b: (4, 4, 1, 0, 5, b.p_tape, None, b.p_out, None, None), 0, "NULL array")
    _add(NODEV_CASES, s, lambda b: (4, 4, 1, 0, 5, b.p_tape, b.p_y, b.p_out, None, None), 0, NODEV)

    # CondatChambollePock2_TV: every refusal marks every image's row, except batch < 0
    for s, host in (("proxtv_CP2_TV_dev_" + t, False), ("proxtv_CP2_TV_batched_" + t, True)):
        tail = (lambda b: (b.p_info,)) if host else (lambda b: (b.p_info, None))
        _add(ARG_CASES, s, lambda b, tail=tail: (4, 4, 3, 0, b.p_y, 0.1, b.p_out, 3, 10) + tail(b), 0,
             "Algorithm parameter has an invalid value", ALL3)
        _add(ARG_CASES, s, lambda b, tail=tail: (4, 4, -1, 0, b.p_y, 0.1, b.p_out, 0, 10) + tail(b), 0, "invalid shape (need batch >= 0)", ROW0)
        _add(ARG_CASES, s, lambda b, tail=tail: (4, 4, 0, 0, b.p_y, 0.1, b.p_out, 0, 10) + tail(b), 1, None)
        _add(ARG_CASES, s, lambda b, tail=tail: (0, 4, 3, 0, b.p_y, 0.1, b.p_out, 0, 10) + tail(b), 0,
             "invalid shape (need 1 <= M, N < 2^31)", ALL3)
        _add(ARG_CASES, s, lambda b, tail=tail: (4, 4, 3, 0, None, 0.1, b.p_out, 0, 10) + tail(b), 0, "NULL array", ALL3)
        _add(NODEV_CASES, s, lambda b, tail=tail: (4, 4, 3, 1, b.p_y, 0.1, b.p_out, 1, 10) + tail(b), 0, NODEV, ALL3)

    # DR2L1W_TV: single image and batched, device and host arrays
    _add(NODEV_CASES, "proxtv_DR2L1W_TV_dev_" + t, lambda b: (4, 4, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_info, None), 0, NODEV, ROW0)
    for s, host in (("proxtv_DR2L1W_TV_batched_dev_" + t, False), ("proxtv_DR2L1W_TV_batched_" + t, True)):
        tail = (lambda b: (b.p_info,)) if host else (lambda b: (b.p_info, None))
        _add(ARG_CASES, s, lambda b, tail=tail: (4, 4, -1, 0, b.p_y, b.p_w, b.p_w, b.p_out, 5) + tail(b), 0,
             "invalid shape (need batch >= 0)", ROW0)
        _add(NODEV_CASES, s, lambda b, tail=tail: (4, 4, 3, 1, b.p_y, b.p_w, b.p_w, b.p_out, 5) + tail(b), 0, NODEV, ROW0)
    too_small = "tape_bytes smaller than proxtv_DR2L1W_TV_batched_tape_bytes()"
    s = "proxtv_DR2L1W_TV_record_dev_" + t
    _add(ARG_CASES, s, lambda b: (4, 0, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0,
         "invalid shape (need M, N, batch >= 1)", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, b.p_y, None, b.p_w, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, "NULL array", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 16, b.p_info, None), 0, too_small, ROW0)
    _add(NODEV_CASES, s, lambda b: (4, 4, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, NODEV, ROW0)
    s = "proxtv_DR2L1W_TV_batched_record_dev_" + t
    _add(ARG_CASES, s, lambda b: (4, 4, 0, 0, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0,
         "invalid shape (need M, N, batch >= 1)", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, 3, 0, b.p_y, b.p_w, None, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, "NULL array", ROW0)
    _add(ARG_CASES, s, lambda b: (4, 4, 3, 0, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 16, None, None), 0, too_small)
    _add(NODEV_CASES, s, lambda b: (4, 4, 3, 1, b.p_y, b.p_w, b.p_w, b.p_out, 5, b.p_tape, 1 << 16, b.p_info, None), 0, NODEV, ROW0)
    s = "proxtv_DR2L1W_TV_vjp_dev_" + t
    _add(ARG_CASES, s, lambda b: (0, 4, 5, b.p_tape, b.p_y, b.p_out, None, None, None), 0, "invalid shape (need M, N, batch >= 1)")
    _add(ARG_CASES, s, lambda b: (4, 4, 5, None, b.p_y, b.p_out, None, None, None), 0, "NULL array")
    _add(NODEV_CASES, s, lambda b: (4, 4, 5, b.p_tape, b.p_y, b.p_out, b.p_out2, b.p_out3, None), 0, NODEV)
    s = "proxtv_DR2L1W_TV_batched_vjp_dev_" + t
    _add(ARG_CASES, s, lambda b: (4, 4, 0, 0, 5, b.p_tape, b.p_y, b.p_out, None, None, None), 0, "invalid shape (need M, N, batch >= 1)")
    _add(ARG_CASES, s, lambda b: (4, 4, 3, 0, 5, b.p_tape, b.p_y, None, None, None, None), 0, "NULL array")
    _add(NODEV_CASES, s, lambda b: (4, 4, 3, 1, 5, b.p_tape, b.p_y, b.p_out, None, None, None), 0, NODEV)

    # N-D solvers: the solve checks the device first; lambdas are scaled only after every refusal
    for solver in ("PD2", "PD", "PDR"):
        _add(NODEV_CASES, "proxtv_%s_TV_dev_%s" % (solver, t),
             lambda b: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 10, None), 0, NODEV, ROW0)
        s = "proxtv_%s_TV_record_dev_%s" % (solver, t)
        rec = lambda b, y=None, lam=None, dims=None, ns=None, nds=2, npen=2, tb=1 << 16: (                  # noqa: E731
            y or b.p_y, lam or b.p_lam, dims or b.p_dims, b.p_out, b.p_info, ns or b.p_ns, nds, npen, 10, b.p_tape, tb, None)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b)[:9] + (None, 1 << 16, None), 0, "NULL array", ROW0)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, nds=0), 0, "invalid dimensions (need 1 <= nds <= 16)", ROW0)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, ns=b.p_nsneg), 0, "invalid dimensions (negative size)", ROW0)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, lam=b.p_neg), 0, "negative penalty", ROW0)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, tb=16), 0, "tape_bytes smaller than proxtv_%s_TV_tape_bytes()" % solver, ROW0)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, dims=b.p_baddims), 0, "invalid penalty dimensions", ROW0)
        if solver == "PD2":
            _add(ARG_CASES, s, lambda b, rec=rec: rec(b, npen=3), 0, "PD2_TV takes 1 or 2 penalty terms", ROW0)
        _add(NODEV_CASES, s, rec, 0, NODEV, ROW0)
        s = "proxtv_%s_TV_vjp_dev_%s" % (solver, t)
        if solver == "PDR":
            vjp = lambda b, ns=None, nds=2: (ns or b.p_ns, nds, 2, b.p_dims, 10, b.p_tape, b.p_y, b.p_out, b.p_lam, None)  # noqa: E731
            vjp_null = lambda b: (b.p_ns, 2, 2, b.p_dims, 10, None, b.p_y, b.p_out, None, None)                              # noqa: E731
        else:
            vjp = lambda b, ns=None, nds=2: (ns or b.p_ns, nds, 2, b.p_dims, 10, 7, b.p_tape, b.p_y, b.p_out, None, None)  # noqa: E731
            vjp_null = lambda b: (b.p_ns, 2, 2, b.p_dims, 10, 7, None, b.p_y, b.p_out, None, None)                           # noqa: E731
        _add(ARG_CASES, s, vjp_null, 0, "NULL array")
        _add(ARG_CASES, s, lambda b, vjp=vjp: vjp(b, nds=17), 0, "invalid dimensions (need 1 <= nds <= 16)")
        _add(NODEV_CASES, s, vjp, 0, NODEV)

    # batched PD_TV / PD2_TV: every refusal marks every item's row
    for solver in ("PD2", "PD"):
        for s, tail in (("proxtv_%s_TV_batched_dev_%s" % (solver, t), (None,)), ("proxtv_%s_TV_batched_%s" % (solver, t), ())):
            _add(NODEV_CASES, s, lambda b, tail=tail: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 3, 10) + tail, 0, NODEV, ALL3)
        s = "proxtv_%s_TV_batched_record_dev_%s" % (solver, t)
        rec = lambda b, y=None, lam=None, nds=2, batch=3, tb=1 << 16: (                                     # noqa: E731
            y or b.p_y, lam or b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, nds, 2, batch, 10, b.p_tape, tb, None)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b)[:10] + (None, 1 << 16, None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, batch=0), 0, "invalid batch (need batch >= 1)")
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, nds=0), 0, "invalid dimensions (need 1 <= nds <= 16)", ALL3)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, lam=b.p_neg), 0, "negative penalty", ALL3)
        _add(ARG_CASES, s, lambda b, rec=rec: rec(b, tb=16), 0, "tape_bytes smaller than proxtv_%s_TV_batched_tape_bytes()" % solver, ALL3)
        _add(NODEV_CASES, s, rec, 0, NODEV, ALL3)
        s = "proxtv_%s_TV_batched_vjp_dev_%s" % (solver, t)
        vjp = lambda b, ns=None, nds=2, batch=3: (ns or b.p_ns, nds, 2, b.p_dims, batch, 10, b.p_tape, b.p_y, b.p_out, None, None)  # noqa: E731
        _add(ARG_CASES, s, lambda b: (None, 2, 2, b.p_dims, 3, 10, b.p_tape, b.p_y, b.p_out, None, None), 0, "NULL array")
        _add(ARG_CASES, s, lambda b, vjp=vjp: vjp(b, batch=0), 0, "invalid batch (need batch >= 1)")
        _add(ARG_CASES, s, lambda b, vjp=vjp: vjp(b, nds=0), 0, "invalid dimensions (need 1 <= nds <= 16)")
        _add(NODEV_CASES, s, vjp, 0, NODEV)

_add(NODEV_CASES, "proxtv_PD_TV_f32", lambda b: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 10), 0, NODEV, ROW0)

# the reference's drop-in symbols
for s in ("hybridTautString_TV1", "TV1D_denoise_tautstring", "dp", "SolveTVConvexQuadratic_a1_nw"):
    if s in ("dp", "SolveTVConvexQuadratic_a1_nw"):
        _add(NODEV_CASES, s, lambda b: (8, b.p_y, 0.1, b.p_out), None, NODEV)
    elif s == "TV1D_denoise_tautstring":
        _add(NODEV_CASES, s, lambda b: (b.p_y, b.p_out, 8, 0.1), None, NODEV)
        _add(ARG_CASES, s, lambda b: (b.p_y, b.p_out, 8, -0.1), None, None)
    else:
        _add(NODEV_CASES, s, lambda b: (b.p_y, 8, 0.1, b.p_out), None, NODEV)
_add(NODEV_CASES, "hybridTautString_TV1_custom", lambda b: (b.p_y, 8, 0.1, b.p_out, 0.0), None, NODEV)
_add(NODEV_CASES, "TV1D_denoise", lambda b: (b.p_y, b.p_out, 8, 0.1), None, NODEV)
_add(ARG_CASES, "TV1D_denoise", lambda b: (b.p_y, b.p_out, 0, 0.1), None, None)
_add(NODEV_CASES, "classicTautString_TV1", lambda b: (b.p_y, 8, 0.1, b.p_out), 1, NODEV)
_add(NODEV_CASES, "linearizedTautString_TV1", lambda b: (b.p_y, 0.1, b.p_out, 8), 1, NODEV)
_add(NODEV_CASES, "tautString_TV1_Weighted", lambda b: (b.p_y, b.p_w, b.p_out, 8), 1, NODEV)
_add(NODEV_CASES, "SolveTVConvexQuadratic_a1", lambda b: (8, b.p_y, b.p_w, b.p_out), None, NODEV)
_add(NODEV_CASES, "PN_TV1", lambda b: (b.p_y, 0.1, b.p_out, b.p_info, 8, 0.0, None), 0, NODEV, ROW0)
_add(NODEV_CASES, "PN_TV1_Weighted", lambda b: (b.p_y, b.p_w, b.p_out, b.p_info, 8, 0.0, None), 0, NODEV, ROW0)
_add(ARG_CASES, "TV", lambda b: (b.p_y, 0.1, b.p_out, b.p_info, 8, 0.5, None), 0, "TV only works for norms p >= 1", ROW0, "TVopt")
_add(ARG_CASES, "TV", lambda b: (b.p_y, 0.1, b.p_out, b.p_info, 8, 2.0, None), 0, "only p = 1 (TV-L1) is implemented on the GPU path", ROW0,
     "TVopt")
_add(NODEV_CASES, "TV", lambda b: (b.p_y, 0.1, b.p_out, b.p_info, 8, 1.0, None), 0, NODEV, ROW0, "TVopt")
_add(ARG_CASES, "DR2_TV", lambda b: (4, 4, b.p_y, 0.1, 0.1, 2.0, 1.0, b.p_out, 1, 5, b.p_info), 0,
     "only p = 1 (TV-L1) penalties are implemented on the GPU path", ROW0)
_add(NODEV_CASES, "DR2_TV", lambda b: (4, 4, b.p_y, 0.1, 0.1, 1.0, 1.0, b.p_out, 1, 5, b.p_info), 0, NODEV, ROW0)
_add(NODEV_CASES, "DR2L1W_TV", lambda b: (4, 4, b.p_y, b.p_w, b.p_w, b.p_out, 1, 5, b.p_info), 0, NODEV, ROW0)
_add(ARG_CASES, "CondatChambollePock2_TV", lambda b: (4, 4, b.p_y, 0.1, b.p_out, 3, 10, b.p_info), 0,
     "Algorithm parameter has an invalid value", ROW0, "Condat2_TV")
_add(NODEV_CASES, "CondatChambollePock2_TV", lambda b: (4, 4, b.p_y, 0.1, b.p_out, 0, 10, b.p_info), 0, NODEV, ROW0, "Condat2_TV")
for s in ("PD2_TV", "PD_TV", "PDR_TV"):
    _add(NODEV_CASES, s, lambda b: (b.p_y, b.p_lam, None, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 1, 10), 0, NODEV, ROW0)

# the lane engine's hooks: no stdout line, and proxtv_last_error() only for a CUDA error
_add(NODEV_CASES, "proxtv_lane_prox_dev_f64", lambda b: (0, b.p_y, None, None, b.p_out, 4, 64, 1, 0.1, None), 0, None)
_add(NODEV_CASES, "proxtv_lane_prox2_dev_f64", lambda b: (0, b.p_y, None, None, b.p_out, b.p_out2, 4, 64, 1, 0.1, None), 0, None)
_add(NODEV_CASES, "proxtv_lane_prox_dev_f32", lambda b: (0, b.p_y, None, None, b.p_out, 4, 64, 1, 0.1, None), 0, None)


@pytest.mark.parametrize("sym,args,rc,msg,info,fn", ARG_CASES)
def test_argument_refusals(capfd, sym, args, rc, msg, info, fn):
    _check(capfd, sym, args, rc, msg, info, fn)


@pytest.mark.skipif(HAS_DEVICE, reason="a CUDA device is present")
@pytest.mark.parametrize("sym,args,rc,msg,info,fn", NODEV_CASES)
def test_no_device_refusals(capfd, sym, args, rc, msg, info, fn):
    _check(capfd, sym, args, rc, msg, info, fn)


def test_tape_bytes_refuse_with_zero(capfd):
    """The tape-size queries answer 0 for arguments the record entry points refuse, and write no message."""
    lib = proxtv_b200.load()
    canary = _canary(lib)
    capfd.readouterr()
    ns = np.array([4, 4], np.int32); p = ns.ctypes.data
    assert lib.proxtv_DR2_TV_tape_bytes(4, 4, 0, 5) == 0
    assert lib.proxtv_DR2L1W_TV_batched_tape_bytes(4, 4, 0, 5) == 0
    for f in (lib.proxtv_PDR_TV_tape_bytes, lib.proxtv_PD_TV_tape_bytes, lib.proxtv_PD2_TV_tape_bytes):
        assert f(None, 2, 2, 10) == 0 and f(p, 0, 2, 10) == 0 and f(p, 2, 0, 10) == 0
    assert lib.proxtv_PD2_TV_tape_bytes(p, 2, 3, 10) == 0
    for f in (lib.proxtv_PD_TV_batched_tape_bytes, lib.proxtv_PD2_TV_batched_tape_bytes):
        assert f(None, 2, 2, 3, 10) == 0 and f(p, 2, 2, 0, 10) == 0 and f(p, 0, 2, 3, 10) == 0
    assert lib.proxtv_DR2_TV_tape_bytes(4, 4, 1, 5) > 0 and lib.proxtv_DR2L1W_TV_tape_bytes(4, 4, 5) > 0
    assert _lib.last_error() == canary and capfd.readouterr().out == ""


# ---- refusals that only a device reaches: the N-D and batched solves check the device before their arguments ----
GPU_CASES = []
for t in ("f64", "f32"):
    for solver in ("PD2", "PD", "PDR"):
        _add(GPU_CASES, "proxtv_%s_TV_dev_%s" % (solver, t),
             lambda b: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 0, 2, 10, None), 0, "invalid dimensions", ROW0)
    for solver in ("PD2", "PD"):
        for s, tail in (("proxtv_%s_TV_batched_dev_%s" % (solver, t), (None,)), ("proxtv_%s_TV_batched_%s" % (solver, t), ())):
            _add(GPU_CASES, s, lambda b, tail=tail: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 0, 2, 3, 10) + tail, 0,
                 "invalid dimensions", ALL3)
            _add(GPU_CASES, s, lambda b, tail=tail: (None, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 3, 10) + tail, 0,
                 "NULL array", ALL3)
            _add(GPU_CASES, s, lambda b, tail=tail: (b.p_y, b.p_lam, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 0, 10) + tail, 0,
                 "invalid batch (need batch >= 1)")
for s in ("PD2_TV", "PD_TV", "PDR_TV"):
    _add(GPU_CASES, s, lambda b: (b.p_y, b.p_lam, b.p_w, b.p_dims, b.p_out, b.p_info, b.p_ns, 2, 2, 1, 10), 0,
         "only p = 1 (TV-L1) penalty terms are implemented on the GPU path", ROW0)
_add(GPU_CASES, "proxtv_DR2L1W_TV_batched_dev_f64", lambda b: (4, 4, 3, 0, None, b.p_w, b.p_w, b.p_out, 5, b.p_info, None), 0,
     "NULL array", ROW0)
_add(GPU_CASES, "proxtv_DR2L1W_TV_batched_f32", lambda b: (4, 4, 3, 0, b.p_y, b.p_w, b.p_w, None, 5, b.p_info), 0, "NULL array", ROW0)


@pytest.mark.gpu
@pytest.mark.parametrize("sym,args,rc,msg,info,fn", GPU_CASES)
def test_device_refusals(capfd, sym, args, rc, msg, info, fn):
    _check(capfd, sym, args, rc, msg, info, fn)


@pytest.mark.gpu
def test_empty_dr2_answers(capfd):
    """DR2_TV() reports the iterations it would have run for an empty image, proxtv_DR2_TV_dev_* the 0 it did; both return 0."""
    lib = proxtv_b200.require_device()
    b = Bufs()
    assert lib.DR2_TV(0, 4, b.p_y, 0.1, 0.1, 1.0, 1.0, b.p_out, 1, 0, b.p_info) == 0
    assert list(b.info[:3]) == [35, INFO0, 0]
    b = Bufs()
    assert lib.proxtv_DR2_TV_batched_f64(4, 4, 0, b.p_y, 0.1, 0.1, b.p_out, 7, b.p_info) == 0
    assert list(b.info[:3]) == [7, INFO0, 0]
    b = Bufs()
    assert lib.proxtv_DR2_TV_dev_f64(0, 4, 1, 0, None, 0.1, 0.1, None, 0, b.p_info, None) == 0
    assert b.info[0] == 0 and b.info[2] == 0
    assert np.all(b.out == -7.0)
