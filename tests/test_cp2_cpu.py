"""CPU tests of CondatChambollePock2_TV (tv1_2d's 'condat', 'chambolle-pock' and 'chambolle-pock-acc'): the port (tests/cp2_port.c)
against the reference's own results (tests/golden/cp2_checks.npz), its length-1 deviation, and the argument checks of the
Python surface and the C ABI, which refuse before any device is needed."""
import os
import sys

import numpy as np
import pytest

import proxtv_b200
from proxtv_b200 import _lib

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import cp2_port as port  # noqa: E402
import make_cp2_checks as CP  # noqa: E402


@pytest.fixture(scope="module")
def cp2chk():
    return np.load(CP.PATH)


def test_port_matches_reference_digests(cp2chk):
    n = 0
    for key, Y, lam, alg, maxit in CP.cases():
        X, info = port.cp2_tv(Y, lam, alg, maxit)
        assert np.array_equal(CP.digest(X), cp2chk[key + "_digest"]), key
        assert info[0] == cp2chk[key + "_iters"] and info[2] == 0, key
        n += 1
    assert n * 2 == len(cp2chk.files)


def test_port_stop_rule_facts(cp2chk):
    """Constant and all-zero images stop after one iteration; the two-level block image at lam = 10 runs all 2500; the accelerated
    rule at lam = 0 (gamma = inf) stops after 3 iterations."""
    for alg in CP.ALGS:
        assert cp2chk["const_a%d_iters" % alg] == 2 and cp2chk["zero_a%d_iters" % alg] == 2
        assert cp2chk["block_a%d_iters" % alg] == 2501
    assert cp2chk["s5_a2_l0_m0_iters"] == 4


def test_length_one_deviation():
    """M == 1 or N == 1: the missing difference term is left out of D (the reference reads outside its empty dual array there).  The
    result is then the iteration of one 1D signal: the same bits for a row and for the column holding it, the 1D prox once converged,
    and a single pixel is returned unchanged after one iteration."""
    from oracle import oracle as O
    y = O.gen_cfg2(1, 200, seed=3, block=8)
    for alg in (0, 1, 2):
        row, irow = port.cp2_tv(y, 0.3, alg)
        col, icol = port.cp2_tv(y.T, 0.3, alg)
        assert np.array_equal(row, col.T) and irow[0] == icol[0]
        if alg < 2:
            assert irow[0] == 2501
            assert np.abs(row.ravel() - O.Port().tv1_condat(y.ravel(), 0.3)).max() < 1e-9
    X, info = port.cp2_tv(np.array([[2.5]]), 0.3, 0)
    assert X[0, 0] == 2.5 and info[0] == 2


def test_python_surface_rejects_unimplemented_methods():
    for m in ("kolmogorov", "yang"):
        with pytest.raises(NotImplementedError, match="condat"):
            proxtv_b200.tv1_2d(np.zeros((4, 4)), 0.1, method=m)
    with pytest.raises(AssertionError):
        proxtv_b200.tv1_2d_batched(np.zeros((2, 4, 4)), 0.1, method="pd")


def test_abi_rejects_bad_alg():
    """Checked before anything else, like the reference (src/TV2Dopt.cpp:600-602): message, info[2] = RC_ERROR, return 0, X untouched."""
    lib = proxtv_b200.load()
    Y = np.asfortranarray(np.random.default_rng(0).normal(size=(6, 5))); X = np.full_like(Y, -7.0); info = np.zeros(3)
    assert lib.CondatChambollePock2_TV(6, 5, Y.ctypes.data, 0.1, X.ctypes.data, 3, 0, info.ctypes.data) == 0
    assert info[2] == 3 and np.all(X == -7.0)
    assert _lib.last_error() == "Condat2_TV: Algorithm parameter has an invalid value"
    Yb = np.zeros((3, 6, 5)); Xb = np.zeros_like(Yb); infob = np.zeros(9)
    assert lib.proxtv_CP2_TV_batched_f64(6, 5, 3, 1, Yb.ctypes.data, 0.1, Xb.ctypes.data, -1, 0, infob.ctypes.data) == 0
    assert np.all(infob[2::3] == 3)


@pytest.mark.skipif(proxtv_b200.load().proxtv_device_count() > 0, reason="a CUDA device is present")
def test_fails_loudly_without_device():
    with pytest.raises(proxtv_b200.ProxTVError):
        proxtv_b200.tv1_2d(np.zeros((8, 8)), 0.1, method="condat")
    with pytest.raises(proxtv_b200.ProxTVError):
        proxtv_b200.tv1_2d_batched(np.zeros((2, 8, 8), dtype=np.float32), 0.1, method="chambolle-pock")
