"""CPU tests of the PDR_TV backward pass (DESIGN.md section 13), no GPU needed.

* The host forward (pdr_vjp_emu.forward with the oracle's exact 1D prox) agrees with the oracle's PDR_TV to 1e-12 relative on the
  parity cases of test_gpu_parity.py (1D to 4D, a repeated axis, 5 terms).
* The host restatement (pdr_vjp_emu.backward) is the exact derivative of that forward: gY and the penalty gradients agree with finite
  differences to 1e-6 relative -- element by element on small 1D / 2D / 3D arrays, along random directions on a larger 3D array, for
  1, 2, 3 and 5 terms, a zero penalty (whose derivative is one-sided: the prox is defined for penalties >= 0), and 1, 2, 5 and 35
  iterations.  The caller's penalty ws_i enters as the scaled npen ws_i, so its gradient is npen glam_i.  The unrolled map is
  piecewise linear, so each difference is taken at the largest step from 1e-6 down that holds no kink (test_drw_vjp_cpu.kink_free).
* The tape-driven form of the restatement (backward_from_tapes) equals the pass-driven one bit for bit.
* The torch path's C-order mapping (reversed shape, axis a -> nds + 1 - a) slices the same fibers as the numpy path's Fortran array.
"""
import numpy as np
import pytest

import pdr_vjp_emu as P
import vjp_emu
from test_drw_vjp_cpu import kink_free


def check_close(fd, an, tol=1e-6):
    """max |fd - an| <= tol max |an|, with max |an| taken as at least 1e-2: a penalty can have next to no effect (every fiber one
    segment after many iterations), and then the differences are rounding noise (about 1e-9) around 0."""
    fd, an = np.asarray(fd, dtype=np.float64), np.asarray(an, dtype=np.float64)
    scale = max(np.max(np.abs(an)), 1e-2)
    assert np.max(np.abs(fd - an)) <= tol * scale, (np.max(np.abs(fd - an)) / scale, fd.ravel()[:6], an.ravel()[:6])


@pytest.fixture(scope="module")
def prox(port):
    return P.exact_prox(port)


def volume(shape, seed):
    """Blocks plus noise: generic data (no ties in the input), so the segmentations are locally constant around it."""
    rng = np.random.default_rng(seed)
    B = rng.normal(0, 1, tuple(n // 3 + 1 for n in shape))
    for a, n in enumerate(shape):
        B = np.repeat(B, 3, axis=a).take(np.arange(n), axis=a)
    return B + rng.normal(0, 0.3, shape)


def objective(prox, y, ns, ws, ds, G, maxit):
    return float(np.sum(P.forward(prox, y, ns, ws, ds, maxit)[0] * G))


# 1D / 2D / 3D, 1 / 2 / 3 / 5 terms, a repeated axis, a zero penalty
CASES = [((9,), [0.3], [1]),
         ((5, 6), [0.25, 0.35], [1, 2]),
         ((5, 6), [0.3, 0.0], [1, 2]),
         ((4, 3, 5), [0.2, 0.3, 0.15], [1, 2, 3]),
         ((3, 4, 3), [0.04, 0.02, 0.06, 0.03, 0.05], [1, 2, 3, 1, 2])]
CASE_IDS = ["1d", "2d", "2d-zero", "3d", "3d-5terms"]


@pytest.mark.parametrize("it", [0, 4])
def test_host_forward_equals_oracle(port, prox, it):
    rng = np.random.default_rng(14)
    for shp, ws, ds in [((40, 36), [0.3, 0.2], [1, 2]), ((24, 20, 12), [0.2, 0.2, 0.2], [1, 2, 3]),
                        ((7, 6, 5, 4), [0.3, 0.1, 0.2, 0.4, 0.05], [1, 2, 3, 4, 2]), ((300,), [0.7], [1])]:
        V = np.asfortranarray(rng.normal(size=shp))
        want, _ = port.pdr_tv(V, ws, ds, maxit=it)
        got, passes = P.forward(prox, V.ravel(order="F"), shp, ws, ds, it)
        K = P.MAX_ITERS if it == 0 else it
        assert len(passes) == (K - 1) * len(ws)
        assert np.abs(got - want.ravel(order="F")).max() <= 1e-12 * np.abs(want).max(), (shp, it)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("maxit", [1, 2, 5, 35])
def test_elementwise(prox, case, maxit):
    """Every element of y and every penalty (right derivative at a zero penalty)."""
    ns, ws, ds = case
    y = volume(ns, 11 + maxit).ravel(order="F")
    G = np.random.default_rng(5).normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, maxit)
    gY, glam = P.backward(passes, G, ns, ws, ds, maxit)
    f0 = objective(prox, y, ns, ws, ds, G, maxit)
    fd = np.empty_like(y)
    for e in range(y.size):
        def step(h):
            yh = y.copy(); yh[e] += h
            return objective(prox, yh, ns, ws, ds, G, maxit) - f0
        fd[e] = kink_free(step)
    check_close(fd, gY)
    fw = []
    for i in range(len(ws)):
        def step(h):
            if ws[i] == 0.0 and h < 0:
                return None
            wh = list(ws); wh[i] += h
            return objective(prox, y, ns, wh, ds, G, maxit) - f0
        fw.append(kink_free(step))
    check_close(fw, len(ws) * glam)          # the caller's ws_i is scaled to npen ws_i: its gradient is npen glam_i


@pytest.mark.parametrize("maxit", [2, 5, 35])
def test_directional(prox, maxit):
    """12 x 10 x 8 with 3 terms: random directions in y, and the penalties one at a time."""
    ns, ws, ds = (12, 10, 8), [0.2, 0.3, 0.25], [1, 2, 3]
    y = volume(ns, 3 + maxit).ravel(order="F")
    rng = np.random.default_rng(17)
    G = rng.normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, maxit)
    gY, glam = P.backward(passes, G, ns, ws, ds, maxit)
    f0 = objective(prox, y, ns, ws, ds, G, maxit)
    for _ in range(2):
        V = rng.normal(size=y.size)
        check_close([kink_free(lambda e: objective(prox, y + e * V, ns, ws, ds, G, maxit) - f0)], [np.sum(gY * V)])
    fw = []
    for i in range(3):
        def step(e):
            wh = list(ws); wh[i] += e
            return objective(prox, y, ns, wh, ds, G, maxit) - f0
        fw.append(kink_free(step))
    check_close(fw, 3 * glam)


def test_one_iteration_is_the_mean():
    """K = 1: out = sum_i y / kk, no pass reaches it; gY = sum_i G / kk in the same association."""
    y = volume((6, 5), 1).ravel(order="F")
    G = np.random.default_rng(2).normal(size=y.size)
    out, passes = P.forward(lambda a, *_: a * np.nan, y, (6, 5), [0.3, 0.2, 0.1], [1, 2, 1], 1)
    assert passes == [] and np.array_equal(out, ((0 + y / 3.0) + y / 3.0) + y / 3.0)
    gY, glam = P.backward([], G, (6, 5), [0.3, 0.2, 0.1], [1, 2, 1], 1)
    assert np.array_equal(gY, (G / 3.0 + G / 3.0) + G / 3.0) and np.array_equal(glam, np.zeros(3))


@pytest.mark.parametrize("case", CASES + [((7, 1, 6), [0.3, 0.2, 0.4], [1, 2, 3])], ids=CASE_IDS + ["len1-axis"])
@pytest.mark.parametrize("maxit", [2, 35])
def test_tape_driven_restatement_equals_pass_driven(prox, case, maxit):
    ns, ws, ds = case
    y = np.round(volume(ns, 9) * 4) / 4                     # ties in the input
    y = y.ravel(order="F")
    G = np.random.default_rng(2).normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, maxit)
    tapes = P.pass_tapes(passes, ns, ws, ds)
    for dt in (np.float64, np.float32):
        Gt, pt = G.astype(dt), [X.astype(dt) for X in passes]
        want = P.backward(pt, Gt, ns, ws, ds, maxit)
        got = P.backward_from_tapes(P.pass_tapes(pt, ns, ws, ds) if dt == np.float32 else tapes, Gt, ns, ds, maxit)
        assert got[0].dtype == dt and np.array_equal(got[0], want[0])
        assert np.array_equal(got[1], want[1])


def test_c_order_axis_mapping():
    """A C-ordered array of shape S is the column-major array of reversed(S); axis a of it is axis nds + 1 - a there.  Both slicings
    cut the same fibers (as sets of elements), of the same count and length."""
    from proxtv_b200 import _pdr_c_order
    rng = np.random.default_rng(0)
    for shape in ((7,), (4, 5), (3, 1, 4), (2, 3, 4, 5), (1, 6, 1, 2, 3)):
        A = rng.permutation(int(np.prod(shape))).reshape(shape).astype(np.float64)      # distinct values
        ds = list(range(1, len(shape) + 1))
        ns, dims = _pdr_c_order(shape, ds)
        for a, d in zip(ds, dims):
            gF, gC = P.geom(shape, a), P.geom(ns, d)
            assert gF[:2] == gC[:2], (shape, a)
            fF = vjp_emu.from_flat(A.ravel(order="F"), *gF)
            fC = vjp_emu.from_flat(A.ravel(order="C"), *gC)
            assert np.array_equal(np.array(sorted(map(tuple, fF))), np.array(sorted(map(tuple, fC)))), (shape, a)
