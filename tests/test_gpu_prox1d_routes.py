"""GPU tests (-m gpu) of the batched 1D TV-L1 prox's forward on every route of its dispatch (prox_dispatch.cu), through every entry that
reaches it: the host ABI proxtv_prox_fibers_f64/_f32, the device ABI proxtv_prox_fibers_dev_* on torch tensors (default and side
streams), tv1_1d_batched / tv1w_1d_batched (numpy and torch) and tv1_1d / tv1w_1d.

expected_route() restates the dispatch and the entry points' conditions; each case names its route in its id and, where the library
shows the route, asserts it: proxtv_lane_guard_last, the kernel-class launch counters (gather and scatter count as two elementwise
launches; contiguous and strided scans count in their own classes) and proxtv_long_fiber_last.  One bar per route, by the arithmetic
the route performs:

  chunked, strided (direct or gather + scatter), sequential, long-fiber tiles and their fallback -- the taut-string scan in the storage
  type: bit for bit the sequential Scan<T> (chunk_emu.seq_fibers) on every fiber; float64 also bit for bit the oracle's linearized /
  weighted taut-string on a sample of fibers; float32 also within 4 ulp32(max|x| + max penalty) * sqrt(longest segment) of the float64
  oracle on the float32-rounded input and weights.
  The float32 bar is not a few ulp32(max|x|): the scan's tube heights are of the order of the penalty, and a segment's value is
  refined, with one rounding each time, at every touch along the segment.  Scan<float> run sequentially on the host (what these routes
  must equal bit for bit, so the bar is a property of the inputs, not of the GPU) is up to 700 ulp32(max|x|), about 0.5 ulp32(lam),
  from the oracle for lam = 1e4 on data of magnitude 1..10; and 21.6 ulp32(max|x| + lam) on a 1600-sample flat segment, 10.2 on a
  4000-sample one, at most 3.6 on the other cases.
  lane -- the slope-form scan (in double for float32, rounded once): bit for bit lane_emu.slope_fibers on every fiber; float64 also
  <= 1e-9 relative and the same jumps(., 1e-9) as the oracle on a sample of fibers.
"""
import ctypes as C
import time
import zlib

import numpy as np
import pytest

import chunk_emu
import lane_emu
from conftest import jumps, relerr
from vjp_emu import flat_index

pytestmark = pytest.mark.gpu

# ---- the dispatch, restated ------------------------------------------------------------------------------------------------------
CH, RCP_N = 32, 64                                   # chunk_core.cuh
LF_TL, LF_HL, LF_HR = 8192, 512, 512                 # long_fiber.cu
LF_W = LF_TL + LF_HL + LF_HR
LF_SCRATCH_MIN_LEN = 16384                           # capi.cu: contiguous fibers longer than this get the long-fiber scratch
KC_CONTIG, KC_STRIDED, KC_ELEMENTWISE = 0, 1, 2      # ptv_internal.h, KernelClass


def _ceil(a, b):
    return -(-a // b)


def chunked_contig_ok(isz, weighted, nf, ln):
    """launch_chunked_contig (kernels_chunked.cu) accepts contiguous fibers when their staging fits 200 KiB of shared memory."""
    half = weighted and isz == 8 and _ceil(ln, 16) <= 1024        # 16-sample chunks for weighted float64
    nrows = _ceil(ln, CH)
    lpf = _ceil(ln, 16) if half else nrows
    if lpf > 1024:
        return False
    pade = 16 // isz
    npad = _ceil(ln + (nrows + 1) * pade, pade) * pade
    fpb = min(max(1, (256 if half else 128) // lpf), nf)
    aliased = fpb * lpf <= 2 * RCP_N
    per_fiber = npad * isz * (2 if weighted else 1) + lpf * (12 + (0 if aliased else isz))
    return per_fiber * fpb + RCP_N * 2 * isz + 16 <= 200 * 1024


def chunked_limit(isz, weighted):
    """Longest fiber the chunked contiguous kernel takes (one fiber per call)."""
    lo, hi = 64, 1 << 17
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if chunked_contig_ok(isz, weighted, 1, mid) else (lo, mid - 1)
    return lo


def strided_direct_ok(isz, nf, ln, inc):
    """prox_fibers_chunked_strided / launch_strided: some group width FPB fits (shared memory, threads) and divides nf and inc."""
    sect = 32 // isz
    pade = 16 // isz
    lpf = _ceil(ln, CH)
    per_fiber = (ln + (lpf + 2) * pade) * isz + lpf * (12 + isz)
    for fpb, budgeted in ((4 * sect, True), (2 * sect, True), (sect, True), (sect // 2, False), (sect, False)):
        if budgeted and per_fiber * fpb > 72 * 1024:
            continue
        npad = _ceil(ln + (lpf + 1) * pade, pade) * pade
        smem = fpb * (npad * isz + lpf * (12 + isz)) + RCP_N * 2 * isz + 16
        if smem <= 220 * 1024 and fpb * lpf <= 1024 and inc % fpb == 0 and nf % fpb == 0:
            return True
    return False


def lane_shape_ok(isz, nf, ln, inc):
    """kernels_lane.cu lane_shape_ok: whole slabs and a 16-byte row pitch (the test's buffers are 256-byte aligned)."""
    if inc > 1 and nf % inc != 0:
        return False
    return ln >= 2 and ((ln if inc == 1 else inc) * isz) % 16 == 0


def guard_ok(flat, lam):
    """solver.cu lane_guard: lane only while lam <= kappa * mean |step| over the first 2^18 stored elements (kappa 1 float64, 2
    float32).  Returns (decision, distance of lam from the threshold relative to lam)."""
    ns = min(flat.size, 1 << 18)        # flat: the nf * len elements the entry points hand to the guard
    step = np.abs(np.diff(flat[:ns].astype(np.float64))).sum() / (ns - 1)
    thr = (1.0 if flat.dtype == np.float64 else 2.0) * step
    return bool(step > 0 and lam <= thr), abs(thr - lam) / lam


def guard_runs(weighted, nf, ln, engine, lam):
    """The entry points consult the guard for unweighted calls on >= 1024 fibers of >= 64 samples; it decides only under 'auto'."""
    return engine == "auto" and not weighted and nf >= 1024 and ln >= 64 and lam > 0


def expected_route(dtype, weighted, nf, ln, inc, engine, lam, guard=True):
    """Kernel family prox_fibers_ex uses for a call of the C ABI (either entry): 'lane', 'chunked', 'long-tiles', 'strided-direct',
    'gather-scatter', 'gather-seq' (the gather runs, the contiguous kernel does not fit, the sequential kernel does the scan) or 'seq'.
    guard: the lane guard's decision for the data (only consulted under 'auto').  Whether long-fiber tiles pass their agreement check
    depends on the data: a failed check is the route 'long-fallback', which the caller names."""
    isz = np.dtype(dtype).itemsize
    lam = float(np.asarray(lam, dtype=dtype))
    if (engine == "lane" or (engine == "auto" and guard)) and not weighted and lam > 0 and ln >= 64 and nf >= 1024 \
            and lane_shape_ok(isz, nf, ln, inc):
        return "lane"
    if engine != "seq" and ln >= 2 * CH:
        if inc == 1:
            if chunked_contig_ok(isz, weighted, nf, ln):
                return "chunked"
            if not weighted and ln > LF_SCRATCH_MIN_LEN and ln >= 2 * LF_W and nf * _ceil(ln, LF_TL) <= 65535:
                return "long-tiles"
        elif not weighted:                                        # both entries give strided calls scratch
            if (engine == "chunked-strided" or nf % inc != 0) and strided_direct_ok(isz, nf, ln, inc):
                return "strided-direct"
            if nf % inc == 0:
                return "gather-scatter" if chunked_contig_ok(isz, False, nf, ln) else "gather-seq"
    return "seq"


def expected_launches(route, inc):
    """(contiguous, strided, elementwise) launch counts, None for 'at least one'."""
    if route == "gather-scatter":
        return (0, None, 2)
    if route == "gather-seq":
        return (0, None, 1)
    return (None, 0, 0) if inc == 1 else (0, None, 0)


# ---- data ------------------------------------------------------------------------------------------------------------------------
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
    if kind == "plateau":                                          # noise, a flat third, noise
        X = rng.normal(0, 1, (nf, ln))
        X[:, ln // 3: 2 * ln // 3] = 0.25
        return X
    raise ValueError(kind)


def weights(nf, ln, rng):
    W = rng.uniform(0.05, 1.0, (nf, max(ln - 1, 0)))
    W[rng.random(W.shape) < 0.1] = 0.0
    return W


class Case:
    """One call: entry, dtype, weighted, geometry, engine, data kind, penalty; special: a constructed long-fiber signal."""

    def __init__(self, entry, dtype, weighted, nf, ln, inc, engine, kind, lam, special=None, stream=False):
        self.entry, self.dtype, self.weighted, self.nf, self.ln, self.inc = entry, dtype, weighted, nf, ln, inc
        self.engine, self.kind, self.lam, self.special, self.stream = engine, kind, lam, special, stream
        self.seed = zlib.crc32(repr((entry, np.dtype(dtype).name, weighted, nf, ln, inc, engine, kind, lam, special)).encode())

    def data(self):
        rng = np.random.default_rng(self.seed)
        nf, ln = self.nf, self.ln
        X = make(self.kind, nf, ln, rng)
        marked = []                                                # constructed fibers: always checked against the oracle
        if self.special == "jump-at-tile":                         # a step exactly at a tile boundary 8192 k
            k = (ln // LF_TL) // 2 or 1
            X[:, k * LF_TL:] += 6.0
            marked = [0, nf - 1]
        elif self.special == "plateau-over-overlap":               # one fiber flat across a tile overlap: the whole call falls back
            f = nf // 2
            b = 3 * LF_TL if ln > 4 * LF_TL else LF_TL
            X[f, b - 2000: b + 2000] = 0.7
            marked = [f]
        elif self.special == "segment-across-boundary":           # a segment from well before a tile start to just past the boundary:
            b = 3 * LF_TL                                          # the tiles disagree on it, though the window holds its end (a jump)
            X[:, b - 1500: b + 100] = 4.0
            marked = [0, nf - 1]
        X = X.astype(self.dtype)
        W = weights(nf, ln, rng).astype(self.dtype) if self.weighted else None
        return X, W, marked

    def route(self, X=None):
        guard = True
        if guard_runs(self.weighted, self.nf, self.ln, self.engine, self.lam):
            if X is None:
                X = self.data()[0]
            guard = guard_ok(device_input(X, self.inc)[:self.nf * self.ln], float(np.asarray(self.lam, self.dtype)))[0]
        if self.special in ("plateau-over-overlap", "single-segment", "segment-across-boundary"):
            return "long-fallback"
        return expected_route(self.dtype, self.weighted, self.nf, self.ln, self.inc, self.engine, self.lam, guard)

    def id(self):
        return "%s-%s-%s%s-nf%d-len%d-inc%d-%s-%s-lam%g%s%s" % (
            self.route(), self.entry, np.dtype(self.dtype).name, "-w" if self.weighted else "", self.nf, self.ln, self.inc,
            self.engine, self.kind, self.lam, "-" + self.special if self.special else "", "-stream" if self.stream else "")


def extent(nf, ln, inc):
    return _ceil(nf, inc) * inc * ln


def flat_of(X, inc):
    """The fibers of X (nf, ln) stored under the slicing (nf, ln, inc); positions outside every fiber are NaN."""
    nf, ln = X.shape
    out = np.full(extent(nf, ln, inc), np.nan, dtype=X.dtype)
    out[flat_index(nf, ln, inc)] = X
    return out


def device_input(X, inc):
    """What the library reads: the fibers of X stored under the slicing, -7 outside them (those values must not matter)."""
    return np.nan_to_num(flat_of(X, inc), nan=-7.0)


# ---- the cases -------------------------------------------------------------------------------------------------------------------
F64, F32 = np.float64, np.float32
KINDS = ("blocks", "ties", "const", "ramp", "alt", "plateau", "offset")
LAMS = (0.3, 0.0, 1e-12, 1.0, 1e4, 0.2, 5.0)


def _cases():
    out = []
    # thresholds of the lane engine (nf >= 1024, len >= 64, 16-byte row pitch) and of the chunked kernel (len >= 64)
    for dt in (F64, F32):
        for entry in ("host", "dev"):
            for nf, ln in ((1024, 63), (1024, 64), (1024, 65), (1023, 64)):
                out.append(Case(entry, dt, False, nf, ln, 1, "auto", "blocks", 0.2, stream=entry == "dev"))
        # the chunked kernel's shared-memory limit and one past it, unweighted (then: long-fiber tiles) and weighted (then: sequential)
        for weighted in (False, True):
            lim = chunked_limit(np.dtype(dt).itemsize, weighted)
            for entry in ("host", "dev"):
                for ln in (lim, lim + 1):
                    out.append(Case(entry, dt, weighted, 3, ln, 1, "auto", "blocks", 0.3))
            out.append(Case("host", dt, weighted, 3, lim, 1, "seq", "ties", 1.0))
    # strided fibers: nf a multiple of inc (gather + scatter, lane, or the direct kernel when asked for) and not (direct kernel or
    # sequential; device entry only: the host entry refuses it), weighted (sequential), every engine that changes the route
    i = 0
    for dt in (F64, F32):
        for inc, ln in ((2, 300), (36, 200), (1024, 100)):
            for weighted in (False, True):
                for engine in ("auto", "chunked-strided", "seq"):
                    kind, lam = KINDS[i % len(KINDS)], LAMS[i % len(LAMS)]
                    i += 1
                    out.append(Case("host" if i % 2 else "dev", dt, weighted, 2 * inc, ln, inc, engine, kind, lam, stream=i % 4 == 0))
                    odd = {2: 5, 36: 40, 1024: 1040}[inc]
                    out.append(Case("dev", dt, weighted, odd, ln, inc, engine, kind, lam))
            out.append(Case("dev", dt, False, 2 * inc, 23000 if inc == 2 else 64, inc, "auto", "ties", 1e4))
        # a strided slab too long for the contiguous kernel: the gather runs, then the sequential kernel
        out.append(Case("host", dt, False, 4, chunked_limit(np.dtype(dt).itemsize, False) + 1, 2, "auto", "blocks", 0.3))
    # long fibers: tile edges (2 LF_W, + 1, 2 * 8192 * k + 1), 10^6 samples, batches, a jump on a tile boundary, a fiber that
    # makes the whole call fall back, one segment
    for dt in (F64, F32):
        for entry in ("host", "dev"):
            for ln in (2 * LF_W, 2 * LF_W + 1, 2 * LF_TL * 2 + 1, 2 * LF_TL * 3 + 1):
                out.append(Case(entry, dt, False, 1, ln, 1, "auto", "blocks", 0.3))
            out.append(Case(entry, dt, False, 1, 1_000_000, 1, "auto", "offset", 0.2, stream=entry == "dev"))
            for nf in (1, 3, 40):
                out.append(Case(entry, dt, False, nf, 60000, 1, "auto", "blocks", 0.3))
            out.append(Case(entry, dt, False, 3, 60000, 1, "auto", "blocks", 0.3, special="jump-at-tile"))
            out.append(Case(entry, dt, False, 3, 60000, 1, "auto", "blocks", 0.3, special="plateau-over-overlap"))
            out.append(Case(entry, dt, False, 40, 60000, 1, "auto", "ties", 1.0, special="plateau-over-overlap"))
            out.append(Case(entry, dt, False, 1, 60000, 1, "auto", "blocks", 1e4, special="single-segment"))
            out.append(Case(entry, dt, False, 2, 60000, 1, "auto", "blocks", 0.3, special="segment-across-boundary"))
    # every engine on one shape that every family can take, contiguous and strided
    for dt in (F64, F32):
        for inc in (1, 8):
            for engine in ("auto", "seq", "chunked", "chunked-strided", "lane"):
                out.append(Case("dev", dt, False, 1024, 256, inc, engine, "blocks", 0.2, stream=True))
            out.append(Case("dev", dt, False, 1024, 256, inc, "auto", "ties", 1e4))           # guard says no
    # the Python entries
    for dt in (F64, F32):
        for entry in ("np-batched", "torch-batched"):
            for nf, ln, weighted, kind, lam in ((1024, 64, False, "blocks", 0.2), (7, 1000, False, "ties", 0.0),
                                                (7, 1000, True, "const", 0.0), (3, 40000, False, "blocks", 0.3),
                                                (2, 30000, True, "alt", 0.0), (5, 40, False, "plateau", 1e-12)):
                out.append(Case(entry, dt, weighted, nf, ln, 1, "auto", kind, lam))
    for weighted in (False, True):
        for ln in (5000, 2 * LF_W + 1, 1_000_000):
            out.append(Case("tv1", F64, weighted, 1, ln, 1, "auto", "blocks", 0.3))
    return out


CASES = _cases()
SEEN = {"routes": set(), "lf_hook": set(), "ran": 0, "t0": None}


# ---- running and checking --------------------------------------------------------------------------------------------------------
def _vp(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def run_entry(ptv, case, X, W):
    """The call under test; returns the output as a flat array in the slicing's storage (NaN where no fiber writes)."""
    lib = ptv.load()
    nf, ln, inc, lam, f32 = case.nf, case.ln, case.inc, case.lam, case.dtype == F32
    xf = device_input(X, inc)
    wf = device_input(W, inc) if W is not None else None
    if case.entry == "host":
        out = np.full_like(xf, np.nan)
        fn = lib.proxtv_prox_fibers_f32 if f32 else lib.proxtv_prox_fibers_f64
        assert fn(_vp(xf), _vp(out), nf, ln, inc, lam, _vp(wf)) == 1, ptv._lib.last_error()
        return out
    if case.entry == "np-batched":
        Y = ptv.tv1w_1d_batched(X, W) if W is not None else ptv.tv1_1d_batched(X, lam)
        assert Y.dtype == X.dtype
        return Y.ravel()
    if case.entry == "tv1":
        Y = ptv.tv1w_1d(X[0], W[0]) if W is not None else ptv.tv1_1d(X[0], lam)
        return Y
    import torch
    if case.entry == "torch-batched":
        xt = torch.from_numpy(X).cuda()
        Y = ptv.tv1w_1d_batched(xt, torch.from_numpy(W).cuda()) if W is not None else ptv.tv1_1d_batched(xt, lam)
        assert Y.dtype == xt.dtype
        return Y.cpu().numpy().ravel()
    xt = torch.from_numpy(device_input(X, inc)).cuda()
    wt = torch.from_numpy(device_input(W, inc)).cuda() if W is not None else None
    out = torch.full_like(xt, float("nan"))
    fn = lib.proxtv_prox_fibers_dev_f32 if f32 else lib.proxtv_prox_fibers_dev_f64
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    if case.stream:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            assert fn(p(xt), p(out), nf, ln, inc, lam, p(wt), C.c_void_p(s.cuda_stream)) == 1, ptv._lib.last_error()
        s.synchronize()
    else:
        assert fn(p(xt), p(out), nf, ln, inc, lam, p(wt), None) == 1, ptv._lib.last_error()
    return out.cpu().numpy()


def sample_fibers(nf, marked, rng, k=12):
    pick = {0, nf - 1, *marked}
    if nf > k:
        pick |= set(rng.choice(nf, k, replace=False).tolist())
    else:
        pick = set(range(nf))
    return sorted(pick)


def check(port, case, route, X, W, marked, got_flat):
    nf, ln, inc = case.nf, case.ln, case.inc
    idx = flat_index(nf, ln, inc)
    assert got_flat.size == extent(nf, ln, inc)
    got = got_flat[idx]
    outside = np.ones(got_flat.size, bool)
    outside[idx.ravel()] = False
    assert np.isnan(got_flat[outside]).all(), "wrote outside the fibers"
    lam = float(np.asarray(case.lam, case.dtype))
    xf = flat_of(X, inc)
    if route == "lane":
        want = lane_emu.slope_fibers(lane_emu.load(), xf, nf, ln, inc, lam)[idx]
    else:
        want = chunk_emu.seq_fibers(xf, nf, ln, inc, lam, flat_of(W, inc) if W is not None else None)[idx]
    bad = np.nonzero(~np.all(got == want, axis=1))[0]
    assert bad.size == 0, "fibers %s differ from the %s restatement (max |diff| %g)" % (
        bad[:8].tolist(), "slope-form" if route == "lane" else "sequential", np.abs(got[bad] - want[bad]).max())
    rng = np.random.default_rng(case.seed + 1)
    X64 = X.astype(np.float64)
    W64 = W.astype(np.float64) if W is not None else None
    for f in sample_fibers(nf, marked, rng):
        if W is not None:
            ref = port.tv1_weighted(X64[f], W64[f]) if ln > 1 else X64[f]
        else:
            ref = port.tv1_linearized(X64[f], lam)
        if case.dtype == F64:
            if route == "lane":
                assert relerr(got[f], ref) <= 1e-9, f
                assert np.array_equal(jumps(got[f], 1e-9), jumps(ref, 1e-9)), f
            else:
                assert np.array_equal(got[f], ref), f
        elif route != "lane":
            scale = np.abs(X64[f]).max() + (W64[f].max(initial=0.0) if W is not None else lam)
            ulp = float(np.spacing(np.float32(scale)))
            longest = int(np.diff(np.flatnonzero(np.r_[True, ref[1:] != ref[:-1], True])).max())
            err = float(np.abs(got[f].astype(np.float64) - ref).max())
            assert err <= 4 * ulp * np.sqrt(longest), (f, err, ulp, longest)


@pytest.fixture
def lib(ptv):
    L = ptv.load()
    prev = ptv.set_engine("auto")
    yield L
    ptv.set_engine(prev)
    L.proxtv_profile_reset()


@pytest.mark.parametrize("case", CASES, ids=[c.id() for c in CASES])
def test_route(ptv, port, lib, case):
    if SEEN["t0"] is None:
        SEEN["t0"] = time.perf_counter()
    X, W, marked = case.data()
    route = case.route(X)
    ptv.set_engine(case.engine)
    guard_calls = guard_runs(case.weighted, case.nf, case.ln, case.engine, case.lam)
    if guard_calls:
        dec, margin = guard_ok(device_input(X, case.inc)[:case.nf * case.ln], float(np.asarray(case.lam, case.dtype)))
        assert margin > 1e-6, "the data sits on the lane guard's threshold"
    lib.proxtv_profile_reset()
    got = run_entry(ptv, case, X, W)
    ms, launches, spans = (C.c_double * 3)(), (C.c_longlong * 3)(), (C.c_longlong * 3)()
    lib.proxtv_profile_read(ms, launches, spans)
    counts = list(launches)
    if guard_calls:
        assert lib.proxtv_lane_guard_last() == int(dec)
    for have, want, name in zip(counts, expected_launches(route, case.inc), ("contiguous", "strided", "elementwise")):
        assert (have >= 1) if want is None else (have == want), (name, counts, route)
    hook = lib.proxtv_long_fiber_last()
    assert hook == {"long-tiles": 1, "long-fallback": 0}.get(route, -1), (hook, route)
    check(port, case, route, X, W, marked, got)
    SEEN["routes"].add((route, np.dtype(case.dtype).name))
    SEEN["lf_hook"].add(hook)
    SEEN["ran"] += 1


def test_host_entry_refuses_a_partial_slab(ptv):
    """With inc > 1 the host entry stages nf * len elements, which hold the slicing only when nf is a multiple of inc: anything else is
    refused before the device is touched, and nothing is written."""
    lib = ptv.load()
    x = np.arange(40, dtype=np.float64); out = np.full_like(x, np.nan)
    assert lib.proxtv_prox_fibers_f64(_vp(x), _vp(out), 5, 8, 2, 0.5, None) == 0
    assert "nf a multiple of inc" in ptv._lib.last_error() and np.isnan(out).all()
    x32 = x.astype(np.float32); out32 = np.full_like(x32, np.nan)
    assert lib.proxtv_prox_fibers_f32(_vp(x32), _vp(out32), 5, 8, 0, 0.5, None) == 0 and np.isnan(out32).all()


def test_every_route_was_taken():
    """Runs after the cases: every route of the table was taken at least once per dtype, and the long-fiber hook read both 1 and 0."""
    if SEEN["ran"] != len(CASES):
        pytest.skip("only %d of %d route cases ran" % (SEEN["ran"], len(CASES)))
    routes = ("lane", "chunked", "long-tiles", "long-fallback", "strided-direct", "gather-scatter", "gather-seq", "seq")
    missing = [(r, d) for r in routes for d in ("float64", "float32") if (r, d) not in SEEN["routes"]]
    elapsed = time.perf_counter() - SEEN["t0"]
    print("\nroutes taken: %s\nlong-fiber hook values: %s\n%d cases in %.1f s"
          % (sorted(SEEN["routes"]), sorted(SEEN["lf_hook"]), SEEN["ran"], elapsed))
    assert not missing, missing
    assert {0, 1} <= SEEN["lf_hook"]
