"""GPU tests (-m gpu) of the staged row pass's d ring (kernels_lane.cu: DRing), held to the same bit-exact bar as test_gpu_lane.py.

The staged Douglas-Rachford row pass (op 1, LOP_DR_B) keeps d = t - x1 of every landed tile in registers until the drain forms
t' = d + x from it, instead of loading x1 and t again.  The ring is indexed by the absolute tile index, so what these tests pin is
what only that bookkeeping can get wrong: fibers that wrap the ring many times, chunked tasks whose halo tiles are landed but never
drained (and halo 0, where every chunk boundary goes through the repair path, which reads B and C itself), partial last groups,
aliased operand arrays (the solver's first half-iteration passes t as both x1 and t), and whole solves against the drain that
re-reads its operands (the 128-row float64 window, tuning variant 5, has no ring).
"""
import ctypes as C

import numpy as np
import pytest

import lane_emu
import synth_inputs as S
from test_gpu_lane import dyadic, dr_host, expected, first_diff, layout, make

pytestmark = pytest.mark.gpu

DEFAULT_TUNING = (0, 32, -1)


@pytest.fixture(scope="module")
def emu():
    return lane_emu.load()


@pytest.fixture
def lane_lib(ptv):
    lib = ptv.load()
    lib.proxtv_lane_tuning(*DEFAULT_TUNING)
    yield lib
    lib.proxtv_lane_tuning(*DEFAULT_TUNING)


def run_dr_b(lib, A, B, Cc, nf, ln, inc, lam, alias):
    """Op 1 on the GPU; with `alias` B and C are one device buffer (holding Cc)."""
    import torch
    dev = torch.device("cuda")
    tA = torch.from_numpy(A).to(dev); tC = torch.from_numpy(Cc).to(dev)
    tB = tC if alias else torch.from_numpy(B).to(dev)
    X = torch.full((A.size,), float("nan"), dtype=tA.dtype, device=dev)
    p = lambda a: C.c_void_p(a.data_ptr())              # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    fn = lib.proxtv_lane_prox_dev_f32 if A.dtype == np.float32 else lib.proxtv_lane_prox_dev_f64
    ok = fn(1, p(tA), p(tB), p(tC), p(X), nf, ln, inc, float(lam), st)
    torch.cuda.synchronize()
    assert ok == 1, lib.proxtv_last_error()
    return X.cpu().numpy()


def check_dr_b(emu, lib, F, nf, ln, inc, lam, dt, rng, what, alias=False):
    T = np.dtype(dt).type
    A = layout(F, inc).astype(dt)
    Cc = rng.normal(0, 1, A.size).astype(dt)
    B = Cc if alias else rng.normal(0, 1, A.size).astype(dt)
    X = run_dr_b(lib, A, B, Cc, nf, ln, inc, T(lam), alias)
    want, _ = expected(emu, 1, A, B, Cc, nf, ln, inc, T(lam))
    assert np.array_equal(X, want), (what, "first differing (fiber, row)", first_diff(X, want, nf, ln, inc, False))


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_dr_b_aliased_operands(emu, lane_lib, dt):
    """B and C the same array (d = 0 exactly): what the solver's first half-iteration runs, on one slab, a batch of slabs with a
    partial fiber group, a fiber length with a partial last group, and chunked fibers."""
    rng = np.random.default_rng(201)
    for nf, ln, inc in ((64, 512, 64), (108, 1000, 36), (100, 1003, 100), (256, 4096, 128)):
        check_dr_b(emu, lane_lib, make("blocks", nf, ln, rng), nf, ln, inc, 0.2, dt, rng, ("alias", nf, ln, inc), alias=True)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_dr_b_ring_wraps(emu, lane_lib, dt):
    """Fibers of 4096 and 4099 rows (the ring wraps 32 to 64 times per task) as one chunk, as chunks of 512 and 64 rows, the default
    plan, and halo 0 (cold starts at every boundary: repairs), each bit-exact; with halo 0 the repair path must have run."""
    rng = np.random.default_rng(202)
    for ln in (4096, 4099):
        F = make("blocks", 108, ln, rng)
        for clen, halo in ((ln, 32), (512, 32), (64, 32), (0, 32), (0, 0), (512, 0)):
            lane_lib.proxtv_lane_tuning(clen, halo, -1)
            lane_lib.proxtv_lane_stats(1)
            check_dr_b(emu, lane_lib, F, 108, ln, 36, 0.2, dt, rng, ("wrap", ln, clen, halo))
            reps = lane_lib.proxtv_lane_stats(1)
            if halo == 0:
                assert reps > 0, (ln, clen, halo)


def _solve_dev(lib, fn, Yt, out, lam, maxit):
    import torch
    info = np.zeros(3)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    M, N = Yt.shape[1], Yt.shape[0]                     # column-major image: the tensor holds its transpose
    fn(M, N, 1, 0, C.c_void_p(Yt.data_ptr()), lam, lam, C.c_void_p(out.data_ptr()), maxit, C.c_void_p(info.ctypes.data), st)
    torch.cuda.synchronize()
    assert info[2] == 0, lib.proxtv_last_error()
    return out.cpu().numpy(), info


def test_dr2_4096_ring_equals_rereading_drain(ptv, engine_lane):
    """The config-2 solve (4096 x 4096 float64, lambda 0.2, 35 iterations + final projection, staged schedule) with the d ring
    (default tuning) and with tuning variant 5 (128-row window: the drain re-reads x1 and t): bit for bit, iterations included.  Each
    call writes another output buffer, so neither replays the other's captured graph."""
    import torch
    lib = ptv.load()
    Y = S.gen_cfg2(4096, 4096, seed=0)                  # column-major float64
    Yt = torch.from_numpy(np.ascontiguousarray(Y.T)).cuda()
    outs = [torch.empty_like(Yt) for _ in range(2)]
    try:
        lib.proxtv_lane_tuning(*DEFAULT_TUNING)
        ring, info_r = _solve_dev(lib, lib.proxtv_DR2_TV_dev_f64, Yt, outs[0], 0.2, 0)
        lib.proxtv_lane_tuning(0, 32, 5)
        reread, info_f = _solve_dev(lib, lib.proxtv_DR2_TV_dev_f64, Yt, outs[1], 0.2, 0)
    finally:
        lib.proxtv_lane_tuning(*DEFAULT_TUNING)
    assert np.array_equal(info_r, info_f)
    assert np.array_equal(ring, reread), "first differing element %s" % (np.argwhere(ring != reread)[:1].tolist(),)


def test_dr2_f32_ring_equals_host_driver(ptv, engine_lane, emu):
    """Float32 has no form without the ring (its 128-row window holds 16 tiles of 8 single-precision values): a 512 x 384 float32
    solve on dyadic input (a column-major view: the staged schedule) equals the host driver bit for bit."""
    import torch
    Y = dyadic((1, 512, 384), 11, np.float32)
    want = dr_host(emu, Y, 0.375, 4)
    tc = torch.tensor(np.ascontiguousarray(Y[0].T), device="cuda").T
    got = ptv.tv1_2d(tc, 0.375, max_iters=4)
    assert got.stride() == tc.stride()
    assert np.array_equal(got.cpu().numpy(), want[0])


@pytest.fixture
def engine_lane(ptv):
    prev = ptv.set_engine("lane")
    yield
    ptv.set_engine(prev)
