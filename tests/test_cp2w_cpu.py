"""CPU tests of the weighted Condat / Chambolle-Pock 2D TV-L1 prox (tv1w_2d's 'condat' and 'chambolle-pock', proxtv_CP2W_TV_*,
DESIGN.md section 15.1).  The reference has no weighted primal-dual solver, so its port (tests/cp2w_port.c) is pinned two ways: with
every weight equal to lambda it is the unweighted port (tests/cp2_port.c, itself pinned to the reference's digests) bit for bit, and it
reaches DR2L1W_TV's objective on random problems.  Also: the column-separable case against the weighted 1D prox, the length-1 rule, the
Python surface's checks and the C ABI's refusals, which need no device."""
import os
import sys

import numpy as np
import pytest

import proxtv_b200
from oracle import oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import cp2_port  # noqa: E402
import cp2w_port as port  # noqa: E402
import make_cp2_checks as CP  # noqa: E402
from test_capi_refusals_cpu import HAS_DEVICE, NODEV, _check  # noqa: E402


def objective(x, y, w1, w2):
    """1/2 ||x - y||^2 + sum w1 |x(i+1, j) - x(i, j)| + sum w2 |x(i, j+1) - x(i, j)|."""
    return 0.5 * np.sum((x - y) ** 2) + np.sum(w1 * np.abs(np.diff(x, axis=0))) + np.sum(w2 * np.abs(np.diff(x, axis=1)))


def test_constant_weights_are_the_unweighted_port():
    """Every fixture case with alg 0 or 1: maps equal to lambda give cp2_port's result bit for bit, iteration count included."""
    n = 0
    for key, Y, lam, alg, maxit in CP.cases():
        if alg == 2:
            continue
        M, N = Y.shape
        want, winfo = cp2_port.cp2_tv(Y, lam, alg, maxit)
        got, ginfo = port.cp2w_tv(Y, np.full((M - 1, N), lam), np.full((M, N - 1), lam), alg, maxit)
        assert np.array_equal(got, want), key
        assert ginfo[0] == winfo[0] and ginfo[2] == 0, key
        n += 1
    assert n == 186


def random_problem(rng):
    """prox_tv_test.py's cross-method problem (sizes 10-29, y = 100 N(0, 1)) with per-edge weights in [0, 20), about 10 % exactly 0."""
    M, N = int(rng.integers(10, 30)), int(rng.integers(10, 30))
    y = 100 * rng.normal(size=(M, N))
    w1 = 20 * rng.random((M - 1, N)); w2 = 20 * rng.random((M, N - 1))
    w1[rng.random(w1.shape) < 0.1] = 0.0; w2[rng.random(w2.shape) < 0.1] = 0.0
    return y, w1, w2


def test_objective_no_worse_than_dr2l1w():
    """20 seeded problems, maxit 5000 for both: the primal-dual result's objective is no worse than DR2L1W_TV's (observed: lower by
    7e-15 to 3.3e-14 relative on every problem, both algs) and the two results agree to 1e-8 (observed max |x_cp - x_dr| 2.3e-10)."""
    P = O.Port()
    rng = np.random.default_rng(151)
    for k in range(20):
        y, w1, w2 = random_problem(rng)
        xd, _ = P.dr2l1w_tv(y, w1, w2, maxit=5000)
        od = objective(xd, y, w1, w2)
        for alg in (0, 1):
            xc, info = port.cp2w_tv(y, w1, w2, alg, 5000)
            oc = objective(xc, y, w1, w2)
            assert oc <= od * (1 + 1e-12), (k, alg, oc, od)
            assert np.abs(xc - xd).max() < 1e-8, (k, alg, np.abs(xc - xd).max())
            assert 2 < info[0] <= 5001


def test_zero_row_weights_separate_the_columns():
    """w_row = 0 disconnects the columns: each column of the result is the weighted 1D prox of that column with its own w_col weights
    (observed max difference 9.7e-13 at the default 2500 iterations)."""
    P = O.Port()
    rng = np.random.default_rng(7)
    for k in range(5):
        M, N = int(rng.integers(10, 31)), int(rng.integers(3, 8))
        y = rng.normal(size=(M, N)); w1 = rng.random((M - 1, N)); w2 = np.zeros((M, N - 1))
        for alg in (0, 1):
            x, _ = port.cp2w_tv(y, w1, w2, alg)
            for j in range(N):
                assert np.abs(x[:, j] - P.tv1_weighted(y[:, j], w1[:, j])).max() < 1e-11, (k, alg, j)


def test_length_one_symmetry():
    """M == 1 or N == 1: a row with weights w and the column holding it with the same weights give the same bits and iteration count,
    the weighted 1D prox once converged; a single pixel is returned unchanged after one iteration."""
    P = O.Port()
    y = O.gen_cfg2(1, 200, seed=3, block=8)
    w = np.random.default_rng(3).uniform(0.0, 0.6, 199)
    for alg in (0, 1):
        row, irow = port.cp2w_tv(y, np.zeros((0, 200)), w[None, :], alg)
        col, icol = port.cp2w_tv(y.T, w[:, None], np.zeros((200, 0)), alg)
        assert np.array_equal(row, col.T) and irow[0] == icol[0]
        assert np.abs(row.ravel() - P.tv1_weighted(y.ravel(), w)).max() < 1e-9
    X, info = port.cp2w_tv(np.array([[2.5]]), np.zeros((0, 1)), np.zeros((1, 0)), 0)
    assert X[0, 0] == 2.5 and info[0] == 2


def test_python_surface_checks():
    """Method, weight-shape and weight-sign checks come before any device work."""
    x, w1, w2 = np.zeros((4, 5)), np.ones((3, 5)), np.ones((4, 4))
    xb, wb1, wb2 = np.zeros((2, 4, 5)), np.ones((2, 3, 5)), np.ones((2, 4, 4))
    for m in ("pd", "nope", "yang"):
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d(x, w1, w2, method=m)
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d_batched(xb, wb1, wb2, method=m)
    with pytest.raises(NotImplementedError, match="gamma = 1 / lambda"):
        proxtv_b200.tv1w_2d(x, w1, w2, method="chambolle-pock-acc")
    with pytest.raises(NotImplementedError, match="gamma = 1 / lambda"):
        proxtv_b200.tv1w_2d_batched(xb, wb1, wb2, method="chambolle-pock-acc")
    for m in ("condat", "chambolle-pock"):
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d(x, w1.T, w2, method=m)                       # the two maps' shapes swapped over
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d(x, w1, np.ones((4, 5)), method=m)
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d(x, -w1, w2, method=m)
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d_batched(xb, wb1[:1], wb2, method=m)
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d_batched(xb, wb1, -wb2, method=m)
        with pytest.raises(AssertionError):
            proxtv_b200.tv1w_2d_batched(x, w1, w2, method=m)                  # 2D input to the batched form


@pytest.mark.skipif(HAS_DEVICE, reason="a CUDA device is present")
def test_fails_loudly_without_device():
    with pytest.raises(proxtv_b200.ProxTVError):
        proxtv_b200.tv1w_2d(np.zeros((8, 8)), np.ones((7, 8)), np.ones((8, 7)), method="condat")
    with pytest.raises(proxtv_b200.ProxTVError):
        proxtv_b200.tv1w_2d_batched(np.zeros((2, 8, 8), np.float32), np.ones((2, 7, 8)), np.ones((2, 8, 7)), method="chambolle-pock")


# ---- the C ABI's refusals (test_capi_refusals_cpu.py's conventions): every refusal marks every image's row, except batch < 0 ----
ALL3 = {2: 3, 5: 3, 8: 3}
ROW0 = {2: 3}
ALG2 = "the weighted solver has no accelerated variant (alg 2); use alg 0 or 1"
ARG_CASES, NODEV_CASES = [], []


def _add(lst, sym, args, rc, msg, info=None):
    lst.append(pytest.param(sym, args, rc, msg, info, id="%s-%d" % (sym, sum(1 for p in lst if p.values[0] == sym))))


for t in ("f64", "f32"):
    for s, host in (("proxtv_CP2W_TV_dev_" + t, False), ("proxtv_CP2W_TV_batched_" + t, True)):
        # args(b, M, N, batch, Y, W1, W2, X, alg) with the buffers of test_capi_refusals_cpu.Bufs; "" = the buffer, None = NULL
        def args(M=4, N=4, batch=3, y="", w1="", w2="", x="", alg=0, host=host):
            def f(b):
                pick = lambda v, d: d if v == "" else v                                         # noqa: E731
                a = (M, N, batch, 0, pick(y, b.p_y), pick(w1, b.p_w), pick(w2, b.p_w), pick(x, b.p_out), alg, 10, b.p_info)
                return a if host else a + (None,)
            return f
        _add(ARG_CASES, s, args(alg=3), 0, "Algorithm parameter has an invalid value", ALL3)
        _add(ARG_CASES, s, args(alg=-1), 0, "Algorithm parameter has an invalid value", ALL3)
        _add(ARG_CASES, s, args(alg=2), 0, ALG2, ALL3)
        _add(ARG_CASES, s, args(batch=1, alg=2), 0, ALG2, ROW0)
        _add(ARG_CASES, s, args(batch=-1), 0, "invalid shape (need batch >= 0)", ROW0)
        _add(ARG_CASES, s, args(batch=0, y=None, w1=None, w2=None, x=None), 1, None)
        _add(ARG_CASES, s, args(M=0), 0, "invalid shape (need 1 <= M, N < 2^31)", ALL3)
        _add(ARG_CASES, s, args(N=0), 0, "invalid shape (need 1 <= M, N < 2^31)", ALL3)
        _add(ARG_CASES, s, args(y=None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, args(x=None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, args(w1=None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, args(w2=None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, args(M=1, w2=None), 0, "NULL array", ALL3)
        _add(ARG_CASES, s, args(N=1, w1=None), 0, "NULL array", ALL3)
        # a map with no edges may be NULL: these reach the device check
        _add(NODEV_CASES, s, args(M=1, w1=None), 0, NODEV, ALL3)
        _add(NODEV_CASES, s, args(N=1, w2=None), 0, NODEV, ALL3)
        _add(NODEV_CASES, s, args(M=1, N=1, w1=None, w2=None, alg=1), 0, NODEV, ALL3)
        _add(NODEV_CASES, s, args(), 0, NODEV, ALL3)


@pytest.mark.parametrize("sym,args,rc,msg,info", ARG_CASES)
def test_abi_argument_refusals(capfd, sym, args, rc, msg, info):
    _check(capfd, sym, args, rc, msg, info)


@pytest.mark.skipif(HAS_DEVICE, reason="a CUDA device is present")
@pytest.mark.parametrize("sym,args,rc,msg,info", NODEV_CASES)
def test_abi_no_device_refusals(capfd, sym, args, rc, msg, info):
    _check(capfd, sym, args, rc, msg, info)
