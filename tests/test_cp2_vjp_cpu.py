"""CPU tests of the converged 2D TV-L1 backward (DESIGN.md section 15.2): the host restatement (tests/cp2_vjp_host.py) against central
finite differences of the float64 primal-dual port, for x, lambda and per-edge weights, alg 0 and 1; the dual-returning port against
the solver ports; and the C ABI's refusals of the record and vjp entry points, which need no device."""
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cp2_port  # noqa: E402
import cp2_vjp_host as H  # noqa: E402
import cp2w_port  # noqa: E402
from test_capi_refusals_cpu import HAS_DEVICE, NODEV, _check  # noqa: E402

EPS = 1e-6
CASES = [("random", 16, 16, 0.3, 0), ("random", 20, 17, 0.6, 1), ("piecewise", 24, 20, 0.2, 0), ("piecewise", 18, 22, 0.4, 1)]


def image(kind, M, N, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.normal(size=(M, N))
    return O.gen_cfg2(M, N, seed=seed + 3, block=6) + 0.05 * rng.normal(size=(M, N))


def prox(Y, W1, W2, alg):
    return H.solve(Y, W1, W2, alg)[0]


def test_dual_port_is_the_solver_ports():
    """X and the iteration count of the dual-returning port are cp2w_port's bit for bit, and with constant maps cp2_port's."""
    for kind, M, N, lam, alg in CASES:
        Y = image(kind, M, N)
        W1, W2 = H.weights(M, N, lam)
        X, _, _, info = H.solve(Y, W1, W2, alg)
        want, winfo = cp2_port.cp2_tv(Y, lam, alg)
        assert np.array_equal(X, want) and info[0] == winfo[0]
        rng = np.random.default_rng(1)
        V1, V2 = rng.uniform(0.0, 0.5, W1.shape), rng.uniform(0.0, 0.5, W2.shape)
        X, _, _, info = H.solve(Y, V1, V2, alg)
        want, winfo = cp2w_port.cp2w_tv(Y, V1, V2, alg)
        assert np.array_equal(X, want) and info[0] == winfo[0]


@pytest.mark.parametrize("kind,M,N,lam,alg", CASES)
def test_jacobian_x_matches_finite_differences(kind, M, N, lam, alg):
    """J v (central differences through the port) equals the cluster projection of v; so does the VJP, J being symmetric."""
    Y = image(kind, M, N)
    W1, W2 = H.weights(M, N, lam)
    X, U1, U2, _ = H.solve(Y, W1, W2, alg)
    f1, f2 = H.fused(X, U1, U2, W1, W2)
    rng = np.random.default_rng(2)
    for _ in range(2):
        v = rng.normal(size=(M, N))
        fd = (prox(Y + EPS * v, W1, W2, alg) - prox(Y - EPS * v, W1, W2, alg)) / (2 * EPS)
        gx = H.vjp(X, f1, f2, v)[0]
        assert np.abs(fd - gx).max() < 1e-6


@pytest.mark.parametrize("kind,M,N,lam,alg", CASES)
def test_lambda_gradient_matches_finite_differences(kind, M, N, lam, alg):
    """<g, dy/dlambda> by central differences in lambda equals glam[0] + glam[1]; per axis, through maps that move one axis only."""
    Y = image(kind, M, N)
    W1, W2 = H.weights(M, N, lam)
    X, U1, U2, _ = H.solve(Y, W1, W2, alg)
    f1, f2 = H.fused(X, U1, U2, W1, W2)
    g = np.random.default_rng(3).normal(size=(M, N))
    glam = H.vjp(X, f1, f2, g)[3]
    d = lambda a, b: np.sum(g * (a - b)) / (2 * EPS)  # noqa: E731
    assert abs(d(prox(Y, W1 + EPS, W2 + EPS, alg), prox(Y, W1 - EPS, W2 - EPS, alg)) - glam.sum()) < 1e-6
    assert abs(d(prox(Y, W1 + EPS, W2, alg), prox(Y, W1 - EPS, W2, alg)) - glam[0]) < 1e-6
    assert abs(d(prox(Y, W1, W2 + EPS, alg), prox(Y, W1, W2 - EPS, alg)) - glam[1]) < 1e-6


@pytest.mark.parametrize("alg", [0, 1])
def test_edge_weight_gradients_match_finite_differences(alg):
    """Per-edge weight gradients on random maps with some zero weights: cut, fused and zero-weight edges of both axes."""
    M, N = 18, 16
    Y = image("piecewise", M, N, seed=4)
    rng = np.random.default_rng(5)
    W1, W2 = rng.uniform(0.1, 0.5, (M - 1, N)), rng.uniform(0.1, 0.5, (M, N - 1))
    W1[rng.random(W1.shape) < 0.1] = 0; W2[rng.random(W2.shape) < 0.1] = 0
    X, U1, U2, _ = H.solve(Y, W1, W2, alg)
    f1, f2 = H.fused(X, U1, U2, W1, W2)
    g = rng.normal(size=(M, N))
    _, gw1, gw2, _ = H.vjp(X, f1, f2, g)
    picks = {1: [tuple(e) for e in np.argwhere(f1)[:3]] + [tuple(e) for e in np.argwhere(~f1 & (W1 > 0))[:4]],
             2: [tuple(e) for e in np.argwhere(f2)[:3]] + [tuple(e) for e in np.argwhere(~f2 & (W2 > 0))[:4]]}
    for axis, edges in picks.items():
        assert edges
        for e in edges:
            Wp = [W1.copy(), W2.copy()]; Wm = [W1.copy(), W2.copy()]
            Wp[axis - 1][e] += EPS; Wm[axis - 1][e] -= EPS
            fd = np.sum(g * (prox(Y, *Wp, alg) - prox(Y, *Wm, alg))) / (2 * EPS)
            assert abs(fd - (gw1 if axis == 1 else gw2)[e]) < 1e-6, (axis, e)


def test_rules_of_the_restatement():
    """A NaN never fuses, a zero weight never fuses, and a lambda that fuses everything gives the image mean's gradient."""
    X = np.array([[1.0, 1.0], [np.nan, 1.0]])
    U1 = np.array([[np.nan, 0.0]]); U2 = np.array([[0.5], [0.5]])
    f1, f2 = H.fused(X, U1, U2, np.array([[0.5, 0.0]]), np.array([[0.5], [0.5]]))
    assert f1.tolist() == [[False, False]] and f2.tolist() == [[True], [False]]      # equal values fuse a clipped edge, NaN ones never
    Y = image("random", 12, 10)
    W1, W2 = H.weights(12, 10, 50.0)
    X, U1, U2, _ = H.solve(Y, W1, W2, 0)
    g = np.random.default_rng(6).normal(size=Y.shape)
    gx, gw1, gw2, glam = H.vjp(X, *H.fused(X, U1, U2, W1, W2), g)
    assert np.allclose(gx, g.mean()) and not gw1.any() and not gw2.any()


# ---- the C ABI: refusals that come before any device work
def _recs(b, fn, alg=0, M=4, N=4, batch=1, Y=True, X=True, tape=True, tb=1 << 16, lam=0.1, W=True):
    y, x, t = (b.p_y if Y else None), (b.p_out if X else None), (b.p_tape if tape else None)
    if "CP2W" in fn:
        w = b.p_w if W else None
        return (M, N, batch, 0, y, w, w, x, alg, 0, b.p_info, t, tb, None)
    return (M, N, batch, 0, y, lam, x, alg, 0, b.p_info, t, tb, None)


REC = ["proxtv_CP2_TV_record_dev_f64", "proxtv_CP2_TV_record_dev_f32", "proxtv_CP2W_TV_record_dev_f64", "proxtv_CP2W_TV_record_dev_f32"]
ALG2 = "the accelerated solver (alg 2) has no converged backward: it does not reach the prox's partition; record with alg 0 or 1"
SHAPE = "invalid shape (need M, N, batch >= 1 and M N < 2^31)"


@pytest.mark.parametrize("fn", REC)
def test_record_refusals(capfd, fn):
    rc_err = {2: 3.0}
    _check(capfd, fn, lambda b: _recs(b, fn, alg=2), 0, ALG2, rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, alg=5), 0, "Algorithm parameter has an invalid value", rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, M=0), 0, SHAPE, rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, batch=0), 0, SHAPE, rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, M=1 << 16, N=1 << 16), 0, SHAPE, rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, Y=False), 0, "NULL array", rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, tape=False), 0, "NULL array", rc_err)
    _check(capfd, fn, lambda b: _recs(b, fn, tb=300), 0, "tape_bytes smaller than proxtv_CP2_TV_tape_bytes()", rc_err)
    if "CP2W" in fn:
        _check(capfd, fn, lambda b: _recs(b, fn, W=False), 0, "NULL array", rc_err)
    else:
        _check(capfd, fn, lambda b: _recs(b, fn, lam=-1.0), 0, "negative penalty", rc_err)
    if not HAS_DEVICE:
        _check(capfd, fn, lambda b: _recs(b, fn), 0, NODEV, rc_err)


VJP = ["proxtv_CP2_TV_vjp_dev_f64", "proxtv_CP2_TV_vjp_dev_f32", "proxtv_CP2W_TV_vjp_dev_f64", "proxtv_CP2W_TV_vjp_dev_f32"]


def _vjps(b, fn, M=4, N=4, batch=1, tape=True, X=True, g=True, gY=True):
    head = (M, N, batch, 0, b.p_tape if tape else None, b.p_y if X else None, b.p_w if g else None, b.p_out if gY else None)
    return head + ((b.p_out2, b.p_out3, None, None) if "CP2W" in fn else (None, None))


@pytest.mark.parametrize("fn", VJP)
def test_vjp_refusals(capfd, fn):
    _check(capfd, fn, lambda b: _vjps(b, fn, N=0), 0, SHAPE)
    _check(capfd, fn, lambda b: _vjps(b, fn, batch=0), 0, SHAPE)
    for which in ("tape", "X", "g", "gY"):
        _check(capfd, fn, lambda b: _vjps(b, fn, **{which: False}), 0, "NULL array")
    if not HAS_DEVICE:
        _check(capfd, fn, lambda b: _vjps(b, fn), 0, NODEV)


def test_tape_bytes():
    import proxtv_b200
    lib = proxtv_b200.load()
    assert lib.proxtv_CP2_TV_tape_bytes(4, 4, 0) == 0
    assert lib.proxtv_CP2_TV_tape_bytes(4, 4, 1) == 256 + 2 * 256
    assert lib.proxtv_CP2_TV_tape_bytes(100, 100, 3) == 256 + 2 * ((30000 // 32 * 4 + 4 + 255) // 256 * 256)


def test_backward_keyword_checks():
    """backward='converged' exists for 'condat' and 'chambolle-pock' only; anything else raises before any device work."""
    import proxtv_b200 as ptv
    x = np.zeros((4, 4))
    for m in ("chambolle-pock-acc", "dr", "pd"):
        with pytest.raises(NotImplementedError, match="converged"):
            ptv.tv1_2d(x, 0.1, method=m, backward="converged")
    for m in ("chambolle-pock-acc", "dr"):
        with pytest.raises(NotImplementedError, match="converged"):
            ptv.tv1_2d_batched(x[None], 0.1, method=m, backward="converged")
    with pytest.raises(NotImplementedError, match="converged"):
        ptv.tv1w_2d(x, np.ones((3, 4)), np.ones((4, 3)), method="dr", backward="converged")
    with pytest.raises(NotImplementedError, match="converged"):
        ptv.tv1w_2d_batched(x[None], np.ones((1, 3, 4)), np.ones((1, 4, 3)), method="dr", backward="converged")
    with pytest.raises(AssertionError):
        ptv.tv1_2d(x, 0.1, method="condat", backward="unrolled")
