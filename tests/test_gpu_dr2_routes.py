"""GPU tests (-m gpu) of the 2D TV-L1 prox's forward, DR2_TV, on every schedule dr2_device (solver.cu) picks, through every entry that
reaches it: numpy tv1_2d / tv1_2d_batched and the raw DR2_TV, torch tv1_2d / tv1_2d_batched in both storage orders (and a view whose
base is not 16-byte aligned), and proxtv_DR2_TV_dev_* on the default and on a side stream; and of the weighted solver DR2L1W_TV
(drw_device) on each of its row and column routes.

expected_schedule() restates dr2_device, dr2_lane_pick and lane_shape_ok (kernels_lane.cu) and, for the plain serial schedule, the
route prox_fibers_ex (prox_dispatch.cu) takes on each pass; the threshold helpers and the lane guard are those of
test_gpu_prox1d_routes.  Each case names its schedule in its id and asserts it where the library shows it: proxtv_lane_guard_last,
and the kernel-class launch counts of one solve, derived from solver.cu (a graph replay adds the counts its capture made, so a replayed
call counts like a fresh one).  How the default reaches each schedule:

  lane / lane-t     'auto' while the guard accepts the data, both penalties are positive and the row pitch suits TMA tiling
                    (column-major: M * itemsize a multiple of 16; row-major, always lane-t: M and N * itemsize both); 'lane', 'lane-t'.
  piped-sparse      'auto', float64, one column-major image with even sides >= 1024 and no side over 96 KiB, whenever the lane
                    engine is out for a reason other than the guard: a zero penalty, or a base that is not 16-byte aligned.  A guard
                    refusal (penalty above the mean step) selects the chunked engine and with it the plain schedule.
  piped-dense       the same image under 'pipelined', or float32 under 'auto' (a side of 2 mod 4 keeps the lane engine out).
  tspace / tpose    'tspace' / 'tpose' on column-major images with both sides >= 64; a side longer than the chunked kernel takes
                    makes the body report rc 2 and the plain schedule runs instead ('tspace-fallback' in the id).
  plain             everything else; its passes go through prox_fibers_ex: 'chunked' (contiguous), 'gather-scatter-sparse' (strided:
                    gather, sparse scan, scatter with the fused output form), 'strided-direct' (engine 'chunked-strided'),
                    'gather-seq' (strided and longer than the chunked kernel) or 'seq'.

Bars, one per arithmetic:
  float64, every schedule  <= 1e-9 relative to the oracle (port.dr2_tv) per image, the same info[0], the same jumps(., 1e-9) on a sample
                           of rows and columns.  Observed: about 1e-13 (the 2*mean sum order is the only difference in the chunked
                           family; the lane engine's slope form adds its own rounding).
  chunked family           every schedule but the lane ones is bit for bit the same as the plain schedule under engine 'chunked' on the
                           same entry and layout: engines seq, chunked, chunked-strided, pipelined, tspace, tpose and 'auto' wherever it
                           does not pick the lane engine.  Each of their prox passes is bit for bit the sequential Scan<T> on every
                           fiber (test_gpu_prox1d_routes), the elementwise Douglas-Rachford forms are the same expressions in the same
                           order, and the constant first pass (prox_const_fibers + broadcast) solves the same constant fiber.
  lane vs chunked          float64: <= 1e-10 relative.
  float32                  against the float64 oracle on the float32-rounded input and penalties: max |diff| <= max(2e-5 max |oracle|,
                           4 (K + 1) ulp32(max |Y| + max(w1, w2))) per image, K the iterations.  Every value the solve forms (t, s,
                           Y - s) is of the order of max |Y| + penalty and each rounding is relative to it, so the error of the output
                           -- a difference of such values -- is absolute in those units, whatever the size of the output; the
                           Douglas-Rachford map is nonexpansive, so the roundings of one iteration are not amplified by the next and
                           add at most linearly.  Observed on an H100: at 35 iterations up to 62 ulp32(max |Y| + w) (1.7 per
                           iteration; 7.1e-6 relative to the output); penalty 5 on unit noise after 2 iterations, an output of
                           max |x| = 5.1e-3 is off by 0.4 ulp32(max |Y| + w) = 4e-7, which is 7.7e-5 relative to the output.
"""
import ctypes as C
import time
import zlib

import numpy as np
import pytest

import synth_inputs as S
from conftest import jumps, relerr
from test_gpu_prox1d_routes import KC_CONTIG, KC_ELEMENTWISE, KC_STRIDED, chunked_contig_ok, chunked_limit, guard_ok, strided_direct_ok

F64, F32 = np.float64, np.float32
MAX_ITERS_DR = 35                                    # ptv_internal.h
PIPE_PARTS = 2                                       # solver.cu, DrPipe::parts
PIPE_MAX_BYTES = 96 * 1024                           # solver.cu: the longest side of a pipelined image
SCHEDULES = ("lane", "lane-t", "piped-sparse", "piped-dense", "tspace", "tpose", "plain")
PASS_ROUTES = ("chunked", "gather-scatter-sparse", "strided-direct", "gather-seq", "seq")
LIM = {F64: chunked_limit(8, False), F32: chunked_limit(4, False)}          # 22326, 32768
WLIM = {F64: chunked_limit(8, True), F32: chunked_limit(4, True)}           # 11162, 21496


# ---- the dispatch, restated ------------------------------------------------------------------------------------------------------
def pass_route(isz, nf, ln, inc, eng):
    """prox_fibers_ex for one unweighted Douglas-Rachford pass (a fused input or output form, so never the lane engine or the long-fiber
    tiles) with the solver's scratch (enough for the sparse strided form)."""
    if eng == "seq" or ln < 64:
        return "seq"
    if inc == 1:
        return "chunked" if chunked_contig_ok(isz, False, nf, ln) else "seq"
    if eng == "chunked-strided" and strided_direct_ok(isz, nf, ln, inc):
        return "strided-direct"
    return "gather-scatter-sparse" if chunked_contig_ok(isz, False, nf, ln) else "gather-seq"


def lane_pitch_ok(isz, M, N, row_major, eng):
    """dr2_lane_pick's shape test (both lane_shape_ok calls and the lane-t pitch rule), buffers 16-byte aligned."""
    lane_t = eng == "lane-t" or row_major
    if M < 2 or N < 2 or (M * isz) % 16:
        return False
    return not lane_t or (N * isz) % 16 == 0


def expected_schedule(dtype, M, N, batch, row_major, engine, w1, w2, aligned=True, guard=True):
    """(schedule, (column-pass route, row-pass route) or None, tspace_fallback) of dr2_device for a call; guard: the lane guard's
    decision for the data (consulted only under 'auto' with a positive penalty)."""
    isz = np.dtype(dtype).itemsize
    w1, w2 = float(np.asarray(w1, dtype)), float(np.asarray(w2, dtype))
    eng = engine
    if eng == "auto" and M * N * batch >= 2 and max(w1, w2) > 0 and not guard:
        eng = "chunked"
    lane_t = eng == "lane-t" or bool(row_major)
    if eng in ("auto", "lane", "lane-t") and w1 > 0 and w2 > 0 and aligned and lane_pitch_ok(isz, M, N, row_major, eng):
        return ("lane-t" if lane_t else "lane"), None, False
    fallback = False
    if eng in ("tspace", "tpose") and not row_major and M >= 64 and N >= 64:
        if chunked_contig_ok(isz, False, N * batch, M) and chunked_contig_ok(isz, False, M * batch, N):
            return eng, None, False
        fallback = True                                  # the body reports rc 2 before anything ran
    if eng in ("auto", "pipelined") and not row_major and batch == 1 and M >= 1024 and N >= 1024 and M % 2 == 0 and N % 2 == 0 \
            and max(M, N) * isz <= PIPE_MAX_BYTES:
        return ("piped-sparse" if eng == "auto" and isz == 8 else "piped-dense"), None, False
    if row_major:
        cols = pass_route(isz, N * batch, M, N, eng)
        rows = pass_route(isz, M * batch, N, 1, eng)
    else:
        cols = pass_route(isz, N * batch, M, 1, eng)
        rows = pass_route(isz, M * batch, N, M, eng)
    return "plain", (cols, rows), fallback


def expected_launches(sched, routes, maxit, engine, row_major, M, N):
    """(contiguous, strided, elementwise) launch counts of one dr2_device solve (solver.cu, dr_tspace.cu, prox_dispatch.cu): the
    means are two elementwise kernels, a gather or a scatter one each; prox_const_fibers, the lane guard and copies count nothing."""
    K = maxit if maxit > 0 else MAX_ITERS_DR
    if sched == "lane":
        return K, K + 1, 2                                # the first column pass is a copy of the constant image
    if sched == "lane-t":
        return K, K + 1, 4                                # + ew_dr_first and the one gather
    if sched in ("tspace", "tpose"):                      # YT gather, means, broadcast; tpose: a gather per column pass, a scatter per row pass
        return K, K + 1, 4 + (2 * K + 1 if sched == "tpose" else 0)
    if sched in ("piped-sparse", "piped-dense"):          # each pass in PIPE_PARTS pieces, a gather / scatter per piece
        return PIPE_PARTS * K, PIPE_PARTS * (K + 1), 3 + 2 * PIPE_PARTS * (K + 1)
    cols, rows = routes
    seq_first = engine == "seq"                           # otherwise the first column pass is the constant fiber + broadcast
    counts = [0, 0, 2 + (0 if seq_first else 1)]
    col_inc = N if row_major else 1
    row_inc = 1 if row_major else M
    for route, inc, passes in ((cols, col_inc, K + (1 if seq_first else 0)), (rows, row_inc, K + 1)):
        cls = KC_CONTIG if route == "chunked" or (route == "seq" and inc == 1) else KC_STRIDED
        counts[cls] += passes
        counts[KC_ELEMENTWISE] += passes * {"gather-scatter-sparse": 2, "gather-seq": 1}.get(route, 0)
    return tuple(counts)


# ---- data ------------------------------------------------------------------------------------------------------------------------
def make_images(kind, batch, M, N, rng):
    if kind == "cfg2":                                   # blocks + noise, the BASELINE config 2 generator
        return np.stack([np.asarray(S.gen_cfg2(M, N, seed=int(rng.integers(1 << 30)), block=16)) for _ in range(batch)])
    if kind == "noise":
        return rng.normal(0, 1, (batch, M, N))
    if kind == "ties":
        return np.round(rng.normal(0, 3, (batch, M, N)))
    raise ValueError(kind)


def stored(X, row_major):
    """The flat array the library reads for images X (B, M, N): each image in row-major (C) or column-major order, back to back."""
    return np.ascontiguousarray(X if row_major else np.transpose(X, (0, 2, 1))).ravel()


ENTRY_LAYOUT = {"np-tv1_2d": 0, "np-batched": 0, "np-DR2_TV": 0, "dev-F": 0, "dev-C": 1,
                "torch-2d-F": 0, "torch-2d-C": 1, "torch-batched-F": 0, "torch-batched-C": 1}
TWO_PENALTIES = ("np-DR2_TV", "dev-F", "dev-C")       # the other entries take one penalty for both axes


class Case:
    def __init__(self, entry, dtype, M, N, batch, engine, w1, w2, kind, maxit=0, stream=False, misalign=False):
        assert entry in TWO_PENALTIES or w1 == w2, entry
        assert batch == 1 or entry in ("np-batched", "torch-batched-F", "torch-batched-C", "dev-F", "dev-C"), entry
        self.entry, self.dtype, self.M, self.N, self.batch, self.engine = entry, dtype, M, N, batch, engine
        self.w1, self.w2, self.kind, self.maxit, self.stream, self.misalign = w1, w2, kind, maxit, stream, misalign
        self.row_major = ENTRY_LAYOUT[entry]
        self.seed = zlib.crc32(repr((np.dtype(dtype).name, M, N, batch, kind, w1, w2)).encode())

    def data(self):
        X = make_images(self.kind, self.batch, self.M, self.N, np.random.default_rng(self.seed))
        return X.astype(self.dtype)

    def lam(self):
        return max(float(np.asarray(self.w1, self.dtype)), float(np.asarray(self.w2, self.dtype)))

    def guard_runs(self):
        return self.engine == "auto" and self.M * self.N * self.batch >= 2 and self.lam() > 0

    def guard(self, X=None):
        if not self.guard_runs():
            return True, np.inf
        X = self.data() if X is None else X
        return guard_ok(stored(X, self.row_major), self.lam())

    def schedule(self, X=None):
        return expected_schedule(self.dtype, self.M, self.N, self.batch, self.row_major, self.engine, self.w1, self.w2,
                                 aligned=not self.misalign, guard=self.guard(X)[0])

    def id(self):
        sched, routes, fb = self.schedule()
        name = sched + ("[%s|%s]" % routes if routes else "") + ("-tspace-fallback" if fb else "")
        return "%s-%s-%s-%dx%dx%d-%s-w%g,%g-%s-it%d%s%s" % (
            name, self.entry, np.dtype(self.dtype).name, self.batch, self.M, self.N, self.engine, self.w1, self.w2, self.kind,
            self.maxit, "-stream" if self.stream else "", "-misaligned" if self.misalign else "")


def _cases():
    out = []
    A = out.append
    for dt in (F64, F32):
        f32 = dt == F32
        # lane engine (guard accepts: 0.2 is well under the mean step of the config 2 images) in both schedules
        A(Case("np-batched", dt, 96, 80, 3, "auto", 0.2, 0.2, "cfg2"))
        A(Case("torch-2d-C", dt, 160, 96, 1, "auto", 0.2, 0.2, "cfg2", maxit=2))
        A(Case("torch-batched-C", dt, 128, 96, 2, "auto", 0.2, 0.2, "cfg2"))
        A(Case("dev-F", dt, 100 if f32 else 102, 64, 1, "auto", 0.2, 0.2, "cfg2", stream=True))
        A(Case("dev-F", dt, 128, 64, 2, "lane-t", 0.3, 0.3, "noise", maxit=1))
        A(Case("np-DR2_TV" if not f32 else "dev-F", dt, 200, 136, 1, "auto", 0.1, 0.25, "cfg2"))
        # pipelined: float64 sparse (a zero penalty, a misaligned base), dense under 'pipelined' / float32 with a side of 2 mod 4
        A(Case("dev-F", dt, 1024, 1024, 1, "pipelined", 5.0, 5.0, "noise", maxit=2, stream=True))
        A(Case("torch-2d-F", dt, 1026, 1030, 1, "auto", 0.2, 0.2, "cfg2", maxit=3))
        A(Case("np-DR2_TV" if not f32 else "dev-F", dt, 1024, 1026, 1, "auto", 0.0, 0.3, "cfg2", maxit=1))
        A(Case("torch-2d-F", dt, 1024, 1024, 1, "auto", 0.2, 0.2, "cfg2", maxit=2, misalign=True))
        A(Case("np-DR2_TV" if not f32 else "dev-F", dt, 1024, 1024, 1, "auto", 0.3, 0.0, "cfg2"))
        # the guard refuses (penalty 5 on unit noise): the plain schedule, even at pipelined sizes
        A(Case("np-tv1_2d" if not f32 else "np-batched", dt, 1024, 1024, 1, "auto", 5.0, 5.0, "noise", maxit=2))
        A(Case("dev-F", dt, 1022, 1024, 1, "pipelined", 0.2, 0.2, "cfg2", maxit=2))           # a side under 1024
        A(Case("dev-F", dt, 1024, 1024, 2, "pipelined", 0.2, 0.2, "cfg2", maxit=1))           # batch > 1
        # transposeless schedules at odd shapes, batches, the 64 threshold and past the chunked fiber limit
        A(Case("dev-F", dt, 97, 131, 3, "tspace", 0.3, 0.3, "cfg2"))
        A(Case("dev-F", dt, 65, 64, 2, "tpose", 0.2, 0.2, "noise", maxit=1))
        A(Case("dev-F", dt, 130, 70, 1, "tpose", 0.25, 0.4, "cfg2", stream=True))
        A(Case("dev-F", dt, 200, 136, 1, "tspace", 5.0, 5.0, "noise", maxit=2))
        A(Case("dev-F", dt, 63, 100, 1, "tspace", 0.3, 0.3, "cfg2"))
        A(Case("dev-C", dt, 97, 131, 1, "tspace", 0.3, 0.3, "cfg2"))                        # row-major: plain
        A(Case("dev-F", dt, LIM[dt] + 74, 64, 1, "tspace", 0.3, 0.3, "noise", maxit=1))
        # plain schedule, row-major (the column pass is the strided one)
        A(Case("torch-2d-C", dt, 481, 321, 1, "auto", 0.2, 0.2, "cfg2", maxit=2))
        A(Case("torch-2d-C", dt, 97, 131, 1, "auto", 0.3, 0.3, "cfg2"))
        A(Case("torch-2d-C", dt, 128, 96, 1, "auto", 0.2, 0.2, "cfg2", misalign=True))
        A(Case("torch-2d-C", dt, 128, 96, 1, "auto", 5.0, 5.0, "noise", maxit=1))
        A(Case("torch-batched-C", dt, 97, 131, 3, "auto", 0.3, 0.3, "ties", maxit=2))
        A(Case("dev-C", dt, 64, 96, 2, "chunked-strided", 0.2, 0.3, "cfg2", stream=True))
        A(Case("dev-C", dt, 40, 70, 2, "seq", 0.3, 0.3, "noise", maxit=2))
        # plain schedule, column-major
        A(Case("np-batched", dt, 97, 131, 3, "auto", 0.3, 0.3, "cfg2"))
        A(Case("torch-batched-F", dt, 97, 131, 3, "auto", 0.3, 0.3, "cfg2", maxit=1))
        A(Case("dev-F", dt, 96, 131, 1, "chunked-strided", 0.3, 0.3, "cfg2"))
        A(Case("dev-F", dt, 90, 70, 1, "seq", 0.3, 0.3, "noise", maxit=2))
        A(Case("np-DR2_TV" if not f32 else "dev-F", dt, 200, 136, 1, "auto", 0.3, 0.0, "cfg2", maxit=2))
        A(Case("dev-F", dt, 200, 136, 1, "auto", 0.0, 0.3, "cfg2", stream=True))
        A(Case("dev-F", dt, 120, 100, 1, "lane", 0.0, 0.2, "noise"))                       # lane forced, a zero weight: plain
        # M or N = 1 or 2, both layouts
        for M, N in ((1, 1), (1, 2), (2, 1), (2, 2), (1, 300), (300, 1), (2, 300), (300, 2)):
            A(Case("dev-F", dt, M, N, 1, "auto", 0.3, 0.3, "noise", maxit=2 if M * N > 4 else 0))
            if M * N > 4:
                A(Case("torch-2d-C", dt, M, N, 1, "auto", 0.3, 0.3, "noise", maxit=1))
        # fibers longer than the chunked kernel takes: sequential, after the gather when strided
        L = LIM[dt] + 74
        A(Case("np-tv1_2d" if not f32 else "np-batched", dt, L, 3, 1, "auto", 0.3, 0.3, "noise", maxit=2))
        A(Case("torch-2d-C", dt, L, 3, 1, "auto", 0.3, 0.3, "noise", maxit=2))
        A(Case("np-batched", dt, 3, L, 1, "auto", 0.3, 0.3, "noise", maxit=1))
        A(Case("torch-2d-C", dt, 3, L, 1, "auto", 0.3, 0.3, "noise", maxit=1))
        A(Case("dev-F", dt, LIM[dt], 4, 1, "auto", 0.3, 0.3, "noise", maxit=1))                # at the limit: chunked
    return out


CASES = _cases()
SEEN = {"pairs": set(), "err": {}, "ran": 0, "t0": None}


# ---- running -----------------------------------------------------------------------------------------------------------------------
def _vp(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _tp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def torch_images(X, row_major, misalign=False):
    """A CUDA tensor (B, M, N) holding X in the given storage order; misalign: a view one element into its buffer."""
    import torch
    B, M, N = X.shape
    flat = torch.from_numpy(stored(X, row_major)).cuda()
    if misalign:
        buf = torch.empty(flat.numel() + 1, dtype=flat.dtype, device=flat.device)
        buf[1:].copy_(flat)
        flat = buf[1:]
    return flat.view(B, M, N) if row_major else flat.view(B, N, M).transpose(1, 2)


def run_entry(ptv, case, X, stream=None):
    """The call under test on images X (B, M, N); returns (result (B, M, N) as float64-or-float32 numpy, info or None)."""
    lib = ptv.load()
    B, M, N = X.shape
    e = case.entry
    if e == "np-tv1_2d":
        return ptv.tv1_2d(np.asfortranarray(X[0]), case.w1, max_iters=case.maxit)[None], None
    if e == "np-batched":
        g = ptv.tv1_2d_batched(X, case.w1, max_iters=case.maxit)
        assert g.dtype == X.dtype
        return g, None
    if e == "np-DR2_TV":
        Y = np.asfortranarray(X[0]); out = np.zeros_like(Y, order="F"); info = np.zeros(3)
        lib.DR2_TV(M, N, _vp(Y), case.w1, case.w2, 1.0, 1.0, _vp(out), 1, case.maxit, _vp(info))
        assert info[2] != 3
        return out[None], info
    import torch
    if e.startswith("torch"):
        t = torch_images(X, case.row_major, case.misalign)
        if e.startswith("torch-2d"):
            g = ptv.tv1_2d(t[0], case.w1, max_iters=case.maxit)[None]
        else:
            g = ptv.tv1_2d_batched(t, case.w1, max_iters=case.maxit)
        assert g.dtype == t.dtype
        return g.cpu().numpy(), None
    Y = torch_images(X, case.row_major)
    out = torch.full_like(Y, float("nan"))
    info = np.zeros(3)
    fn = lib.proxtv_DR2_TV_dev_f32 if case.dtype == F32 else lib.proxtv_DR2_TV_dev_f64
    if case.stream:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn(M, N, B, case.row_major, _tp(Y), case.w1, case.w2, _tp(out), case.maxit, _vp(info), C.c_void_p(s.cuda_stream))
        s.synchronize()
    else:
        fn(M, N, B, case.row_major, _tp(Y), case.w1, case.w2, _tp(out), case.maxit, _vp(info), None)
        torch.cuda.synchronize()
    assert info[2] != 3
    return out.cpu().numpy(), info


def read_launches(lib):
    ms, launches, spans = (C.c_double * 3)(), (C.c_longlong * 3)(), (C.c_longlong * 3)()
    lib.proxtv_profile_read(ms, launches, spans)
    return tuple(launches)


def oracle_images(port, X, w1, w2, maxit):
    """port.dr2_tv on every image of X in float64 (the float32-rounded values for float32 input); (results, info of the last)."""
    outs, info = [], None
    for img in X.astype(np.float64):
        o, info = port.dr2_tv(img, w1, w2, maxit=maxit)
        outs.append(o)
    return np.stack(outs), info


def f32_ok(got, want, X, lam, maxit):
    """The float32 bar (module docstring): (passes, max |diff| in ulp32(max |Y| + lam), relative error)."""
    K = maxit if maxit > 0 else MAX_ITERS_DR
    diff = float(np.abs(got.astype(np.float64) - want).max())
    ulp = float(np.spacing(np.float32(np.abs(X).max() + lam)))
    scale = float(np.abs(want).max())
    return diff <= max(2e-5 * scale, 4 * (K + 1) * ulp), diff / ulp, diff / max(scale, 1e-300)


def note_err(key, err):
    SEEN["err"][key] = max(SEEN["err"].get(key, 0.0), err)


def sample_lines(n, rng, k=8):
    return sorted({0, n - 1, *rng.choice(n, min(k, n), replace=False).tolist()})


@pytest.fixture
def lib(ptv):
    L = ptv.load()
    prev = ptv.set_engine("auto")
    yield L
    ptv.set_engine(prev)
    L.proxtv_profile_reset()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id() for c in CASES])
def test_dr2_route(ptv, port, lib, case):
    if SEEN["t0"] is None:
        SEEN["t0"] = time.perf_counter()
    X = case.data()
    sched, routes, fallback = case.schedule(X)
    dec, margin = case.guard(X)
    assert margin > 1e-3, "the data sits on the lane guard's threshold"
    ptv.set_engine(case.engine)
    lib.proxtv_profile_reset()
    got, info = run_entry(ptv, case, X)
    counts = read_launches(lib)
    if case.guard_runs():
        assert lib.proxtv_lane_guard_last() == int(dec)
    want_counts = expected_launches(sched, routes, case.maxit, case.engine, case.row_major, case.M, case.N)
    assert counts == want_counts, (counts, want_counts, sched, routes)
    assert got.shape == X.shape and np.isfinite(got).all()
    # the chunked family: bit for bit the plain schedule under engine 'chunked' on the same entry; lane: within 1e-10 (float64)
    ptv.set_engine("chunked")
    ref_chunked, _ = run_entry(ptv, case, X)
    if sched in ("lane", "lane-t"):
        if case.dtype == F64:
            for b in range(case.batch):
                assert relerr(got[b], ref_chunked[b]) <= 1e-10, b
    else:
        assert np.array_equal(got, ref_chunked), "differs from the chunked engine (max |diff| %g)" % np.abs(got - ref_chunked).max()
    # the float64 oracle
    w1, w2 = float(np.asarray(case.w1, case.dtype)), float(np.asarray(case.w2, case.dtype))
    want, winfo = oracle_images(port, X, w1, w2, case.maxit)
    if info is not None:
        assert info[0] == winfo[0] and info[2] == winfo[2]
    rng = np.random.default_rng(case.seed + 1)
    key = (sched, np.dtype(case.dtype).name)
    for b in range(case.batch):
        err = relerr(got[b], want[b]) if np.abs(want[b]).max() > 0 else float(np.abs(got[b]).max())
        note_err(key, err)
        for r in routes or ():
            note_err(("plain:" + r, key[1]), err)
        if case.dtype == F64:
            assert err <= 1e-9, (b, err)
            for r in sample_lines(case.M, rng):
                assert np.array_equal(jumps(got[b, r, :], 1e-9), jumps(want[b, r, :], 1e-9)), ("row", b, r)
            for c in sample_lines(case.N, rng):
                assert np.array_equal(jumps(got[b, :, c], 1e-9), jumps(want[b, :, c], 1e-9)), ("col", b, c)
        else:
            ok, ulps, rel = f32_ok(got[b], want[b], X[b], case.lam(), case.maxit)
            assert ok, (b, ulps, rel)
    SEEN["pairs"].add(key)
    if routes:
        SEEN["pairs"].update(("plain:" + r, np.dtype(case.dtype).name) for r in routes)
    if fallback:
        SEEN["pairs"].add(("tspace-fallback", np.dtype(case.dtype).name))
    SEEN["ran"] += 1


def existing_pairs():
    """Every (schedule, dtype) pair dr2_device has, plain's pass routes as 'plain:<route>' and the transposeless rc-2 fallback."""
    pairs = {(s, d) for s in SCHEDULES for d in ("float64", "float32") if (s, d) != ("piped-sparse", "float32")}
    pairs |= {("plain:" + r, d) for r in PASS_ROUTES for d in ("float64", "float32")}
    pairs |= {("tspace-fallback", d) for d in ("float64", "float32")}
    return pairs


def table_pairs():
    pairs = set()
    for c in CASES:
        sched, routes, fb = c.schedule()
        d = np.dtype(c.dtype).name
        pairs.add((sched, d))
        pairs |= {("plain:" + r, d) for r in (routes or ())}
        if fb:
            pairs.add(("tspace-fallback", d))
    return pairs


def test_case_table_reaches_every_schedule():
    """CPU: the case table (restated dispatch, the data's guard decision) reaches every schedule and plain pass route in both dtypes,
    and no case's data sits near the lane guard's threshold.  Keeps the table honest when thresholds move."""
    missing = existing_pairs() - table_pairs()
    assert not missing, sorted(missing)
    for c in CASES:
        assert c.guard()[1] > 1e-3, c.id()


# ---- every engine on one image: the chunked family bit for bit, the lane engine within 1e-10 -------------------------------------------
FAMILY = [
    # (dtype, M, N, batch, row_major, w1, w2, kind, maxit, engines, oracle)
    (F64, 1024, 1024, 1, 0, 0.0, 0.2, "cfg2", 3, None, True),          # auto: piped-sparse
    (F32, 1026, 1030, 1, 0, 0.2, 0.2, "cfg2", 3, None, True),          # auto: piped-dense
    (F64, 97, 131, 3, 1, 0.3, 0.3, "cfg2", 0, None, True),
    (F32, 64, 96, 2, 1, 5.0, 5.0, "noise", 0, None, True),
    (F64, 256, 192, 1, 0, 0.2, 0.2, "cfg2", 0, None, True),            # auto: lane
    (F64, 160, 96, 2, 1, 0.2, 0.2, "cfg2", 2, None, True),             # auto: lane-t
    # the pipelined 96 KiB limit and one past it, the chunked fiber limits: bit-equality only
    (F64, 12288, 1024, 1, 0, 0.0, 0.2, "cfg2", 2, ("auto", "chunked", "pipelined", "tspace"), False),
    (F64, 12290, 1024, 1, 0, 0.0, 0.2, "cfg2", 2, ("auto", "chunked", "pipelined", "tspace"), False),
    (F32, 24576, 1024, 1, 0, 0.2, 0.2, "cfg2", 2, ("auto", "chunked", "pipelined", "tspace"), False),
    (F32, 24578, 1024, 1, 0, 0.2, 0.2, "cfg2", 2, ("auto", "chunked", "pipelined", "tspace"), False),
    (F64, LIM[F64] + 1, 64, 1, 0, 0.3, 0.3, "noise", 2, ("auto", "chunked", "seq", "tspace", "tpose"), False),
    (F32, LIM[F32] + 1, 64, 1, 0, 0.3, 0.3, "noise", 2, ("auto", "chunked", "seq", "tspace", "tpose"), False),
    (F64, 64, LIM[F64] + 1, 1, 1, 0.3, 0.3, "noise", 2, ("auto", "chunked", "chunked-strided", "seq"), False),
]
ALL_ENGINES = ("auto", "seq", "chunked", "chunked-strided", "pipelined", "tspace", "tpose", "lane", "lane-t")


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILY, ids=["%s-%dx%dx%d-%s" % (np.dtype(f[0]).name, f[3], f[1], f[2], "C" if f[4] else "F")
                                             for f in FAMILY])
def test_engines_agree(ptv, port, lib, fam):
    dt, M, N, B, rm, w1, w2, kind, maxit, engines, check_oracle = fam
    case = Case("dev-C" if rm else "dev-F", dt, M, N, B, "auto", w1, w2, kind, maxit)
    X = case.data()
    res, scheds = {}, {}
    for e in engines or ALL_ENGINES:
        case.engine = e
        sched, routes, _ = case.schedule(X)
        ptv.set_engine(e)
        lib.proxtv_profile_reset()
        res[e], info = run_entry(ptv, case, X)
        assert read_launches(lib) == expected_launches(sched, routes, maxit, e, rm, M, N), (e, sched, routes)
        scheds[e] = sched
    base = res["chunked"]
    for e, r in res.items():
        if scheds[e] in ("lane", "lane-t"):
            if dt == F64:
                assert max(relerr(r[b], base[b]) for b in range(B)) <= 1e-10, e
        else:
            assert np.array_equal(r, base), (e, scheds[e], np.abs(r - base).max())
    if check_oracle:
        want, _ = oracle_images(port, X, float(np.asarray(w1, dt)), float(np.asarray(w2, dt)), maxit)
        for b in range(B):
            assert relerr(base[b], want[b]) <= 1e-9 if dt == F64 else f32_ok(base[b], want[b], X[b], case.lam(), maxit)[0], b


# ---- graph replay of the captured schedules ------------------------------------------------------------------------------------------
REPLAY = [("piped-dense", F64, 1024, 1024, 1, "pipelined"), ("piped-sparse", F64, 1024, 1024, 1, "auto"),
          ("piped-dense", F32, 1026, 1030, 1, "auto"), ("tspace", F64, 130, 96, 2, "tspace"), ("tpose", F32, 97, 131, 2, "tpose"),
          ("lane", F64, 128, 96, 2, "auto"), ("lane-t", F32, 128, 96, 2, "lane-t")]


@pytest.mark.gpu
@pytest.mark.parametrize("sched,dt,M,N,B,engine", REPLAY, ids=["%s-%s" % (r[0], np.dtype(r[1]).name) for r in REPLAY])
def test_graph_replay(ptv, lib, sched, dt, M, N, B, engine):
    """A captured schedule replayed with new data in the same buffers, after a change of w, maxit or batch alone, and alternating with
    another shape in the same buffers, gives what a call in buffers of its own gives, bit for bit, and counts the same launches."""
    import torch
    ptv.set_engine(engine)
    w2 = 0.0 if sched == "piped-sparse" else 0.3               # a zero penalty keeps the lane engine out of the sparse schedule
    fn = lib.proxtv_DR2_TV_dev_f32 if dt == F32 else lib.proxtv_DR2_TV_dev_f64
    tdt = torch.float64 if dt == F64 else torch.float32
    cap = (B + 1) * (M + 2) * (N + 2)
    bufs = [(torch.empty(cap, dtype=tdt, device="cuda"), torch.empty(cap, dtype=tdt, device="cuda")) for _ in range(2)]

    def images(seed, b, m, n):
        return make_images("cfg2", b, m, n, np.random.default_rng(seed)).astype(dt)

    def call(k, X, w1, maxit):
        """The solve of X in buffer pair k: (result, launch counts).  The graph is keyed by the buffers, so a call in the other pair
        captures afresh and a call right after one with the same arguments replays."""
        b, m, n = X.shape
        Y, out = bufs[k]
        Y[:b * m * n].copy_(torch.from_numpy(stored(X, 0)))
        out.fill_(float("nan"))
        info = np.zeros(3)
        lib.proxtv_profile_reset()
        fn(m, n, b, 0, _tp(Y), w1, w2, _tp(out), maxit, _vp(info), None)
        torch.cuda.synchronize()
        assert info[2] != 3
        return out[:b * m * n].cpu().numpy(), read_launches(lib)

    def same(a, b):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], (np.nanmax(np.abs(a[0] - b[0])), a[1], b[1])

    X1, X2 = images(1, B, M, N), images(2, B, M, N)
    w1 = 0.25
    sched_run = expected_schedule(dt, M, N, B, 0, engine, w1, w2, guard=guard_ok(stored(X1, 0), max(w1, w2))[0])
    assert sched_run[0] == sched
    r1 = call(0, X1, w1, 3)                                    # capture
    assert r1[1] == expected_launches(sched, None, 3, engine, 0, M, N)
    r2 = call(0, X2, w1, 3)                                    # replay with new data in the same buffers
    r3 = call(0, X2, w1, 3)                                    # and again
    same(r2, call(1, X2, w1, 3))
    same(r3, r2)
    same(r1, call(1, X1, w1, 3))
    # only w, only maxit, only the batch (the batched schedules) or only the data's shape (the single-image ones) changes
    Xb = images(3, B + 1, M, N) if B > 1 else images(3, 1, M + 2, N)
    for w1b, maxit, Xc in ((0.35, 3, X2), (w1, 1, X2), (w1, 3, Xb)):
        call(0, X2, w1, 3)
        changed = call(0, Xc, w1b, maxit)
        same(changed, call(1, Xc, w1b, maxit))
    # two shapes alternating in the same buffers
    Z = images(4, B, M + 2, N + 2)
    solo1, solo2 = call(1, X1, w1, 2), call(1, Z, w1, 2)
    for _ in range(2):
        same(call(0, X1, w1, 2), solo1)
        same(call(0, Z, w1, 2), solo2)


# ---- DR2L1W_TV ---------------------------------------------------------------------------------------------------------------------------
def drw_routes(dtype, M, N, engine):
    """(column route, row route) of drw_device: columns through prox_fibers_ex with per-edge weights (chunked, 16-sample chunks in
    float64, or seq); rows 'fast' (gather + sparse weighted chunked kernel + scatter), 'seq', or 'switch' (the sparse kernel refuses
    on the first iteration and the solve goes on with seq rows)."""
    isz = np.dtype(dtype).itemsize
    cols = "chunked" if engine != "seq" and M >= 64 and chunked_contig_ok(isz, True, N, M) else "seq"
    if engine == "seq" or N < 64:
        rows = "seq"
    else:
        rows = "fast" if chunked_contig_ok(isz, True, M, N) else "switch"
    return cols, rows


def drw_launches(routes, M, maxit):
    K = maxit if maxit > 0 else MAX_ITERS_DR
    cols, rows = routes
    counts = [K + 1, 0, 2]                                    # a column pass per iteration and the final one; the means
    if rows == "fast":
        counts[KC_STRIDED] += K + 1
        counts[KC_ELEMENTWISE] += 1 + 2 * (K + 1)             # the W2 gather once, a gather and a scatter per row pass
    else:
        counts[KC_CONTIG if M == 1 else KC_STRIDED] += K + 1
        counts[KC_ELEMENTWISE] += 2 if rows == "switch" else 0   # the W2 gather and the one gather before the refusal
    return tuple(counts)


DRW = []
for _dt in (F64, F32):
    _W = WLIM[_dt] + 38
    for _M, _N, _maxit in ((200, 150, 0), (40, 300, 2), (_W, 3, 2), (300, 40, 2), (150, 200, 1), (3, _W, 2), (1, 200, 2),
                           (70, 1, 2), (64, 64, 0)):
        DRW.append((_dt, _M, _N, _maxit))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,M,N,maxit", DRW, ids=["%s-%s-%dx%d-it%d" % ("cols-%s-rows-%s" % drw_routes(d, m, n, "auto"),
                                                                         np.dtype(d).name, m, n, it) for d, m, n, it in DRW])
def test_drw_route(ptv, port, lib, dt, M, N, maxit):
    """DR2L1W_TV on each route: seq, chunked and auto bit for bit equal to each other; float64 <= 1e-9 relative to the oracle (and the
    numpy tv1w_2d the same), float32 <= 2e-5 relative to the oracle on the float32-rounded input and weights.  A column and a row of
    the weights are all zero."""
    import torch
    rng = np.random.default_rng(zlib.crc32(repr((np.dtype(dt).name, M, N)).encode()))
    Y = (rng.normal(0, 1, (M, N)) + np.repeat(rng.normal(0, 1, (M, 1)), N, axis=1)).astype(dt)
    W1 = rng.uniform(0.05, 0.6, (M - 1, N)).astype(dt)
    W2 = rng.uniform(0.05, 0.6, (M, N - 1)).astype(dt)
    if W1.size:
        W1[:, N // 2] = 0.0                                    # a column whose edges are all free
    if W2.size:
        W2[M // 2, :] = 0.0                                    # a row likewise
    fn = lib.proxtv_DR2L1W_TV_dev_f32 if dt == F32 else lib.proxtv_DR2L1W_TV_dev_f64
    dev = lambda A: torch.from_numpy(np.ascontiguousarray(A.T)).cuda()     # noqa: E731  column-major storage
    Yd, W1d, W2d = dev(Y), dev(W1), dev(W2)
    res = {}
    for e in ("auto", "chunked", "seq"):
        ptv.set_engine(e)
        out = torch.full_like(Yd, float("nan"))
        info = np.zeros(3)
        lib.proxtv_profile_reset()
        fn(M, N, _tp(Yd), _tp(W1d), _tp(W2d), _tp(out), maxit, _vp(info), None)
        torch.cuda.synchronize()
        assert info[2] != 3 and info[0] == (maxit if maxit > 0 else MAX_ITERS_DR)
        assert read_launches(lib) == drw_launches(drw_routes(dt, M, N, e), M, maxit), e
        res[e] = out.cpu().numpy().T
    assert np.array_equal(res["auto"], res["chunked"]) and np.array_equal(res["auto"], res["seq"]), \
        np.abs(res["auto"] - res["seq"]).max()
    want, winfo = port.dr2l1w_tv(Y.astype(np.float64), W1.astype(np.float64), W2.astype(np.float64), maxit=maxit)
    err = relerr(res["auto"], want)
    note_err(("drw:cols-%s-rows-%s" % drw_routes(dt, M, N, "auto"), np.dtype(dt).name), err)
    if dt == F64:
        assert err <= 1e-9
        ptv.set_engine("auto")
        assert np.array_equal(ptv.tv1w_2d(Y, W1, W2, max_iters=maxit), res["auto"])
    else:
        assert err <= 2e-5


@pytest.mark.gpu
def test_every_schedule_was_taken():
    """Runs last: the GPU run took every (schedule, dtype) pair; prints the largest relative error against the oracle per schedule, plain
    pass route and weighted route, and the time since the first case."""
    if SEEN["ran"] != len(CASES):
        pytest.skip("only %d of %d cases ran" % (SEEN["ran"], len(CASES)))
    print("\nlargest relative error against the oracle:")
    for k in sorted(SEEN["err"]):
        print("  %-32s %-8s %.3g" % (k[0], k[1], SEEN["err"][k]))
    print("%d DR2_TV route cases; %.1f s from the first test of the file to this one" % (SEEN["ran"], time.perf_counter() - SEEN["t0"]))
    missing = existing_pairs() - SEEN["pairs"]
    assert not missing, sorted(missing)
