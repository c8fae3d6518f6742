"""CPU tests of the PD_TV and PD2_TV backward passes (DESIGN.md section 14), no GPU needed.

* The host forward (pd_vjp_emu.forward with the oracle's exact 1D prox, run for the oracle's own iteration count) agrees with the
  oracle's PD_TV / PD2_TV to 1e-12 relative on the parity cases (1D to 4D, a repeated axis, 5 terms; PD2_TV with 1 and 2 terms).
* The host restatement (pd_vjp_emu.backward) is the exact derivative of the K-iteration forward: gY and the penalty gradients agree with
  finite differences to 1e-6 relative -- element by element on small 1D / 2D / 3D arrays with 1, 2, 3 and 5 terms (PD_TV) and 1 and 2
  terms (PD2_TV), a zero penalty (right derivative), K = 1, 2, 5 and 35, and along random directions on a 12 x 10 x 8 array.  K is an
  argument here, so no step can change it.  PD_TV's caller penalty ws_i enters as npen ws_i, so its gradient is npen glam_i; PD2_TV's
  penalties enter as given.  Each difference is taken at the largest step from 1e-6 down that holds no kink
  (test_drw_vjp_cpu.kink_free).
* The tape-driven form of the restatement (backward_from_tapes) equals the pass-driven one bit for bit.
* The tape sizes are computed in 64-bit arithmetic: exact past 2^32 passes, 0 (refused by the record calls) past 2^64 bytes.
"""
import numpy as np
import pytest

import pd_vjp_emu as P
from pdr_vjp_emu import exact_prox
from test_drw_vjp_cpu import kink_free
from test_pdr_vjp_cpu import check_close, volume


@pytest.fixture(scope="module")
def prox(port):
    return exact_prox(port)


def objective(prox, y, ns, ws, ds, G, K, pd2):
    return float(np.sum(P.forward(prox, y, ns, ws, ds, K, pd2)[0] * G))


PARITY = [(False, (40, 36), [0.3, 0.2], [1, 2]), (False, (24, 20, 12), [0.2, 0.2, 0.2], [1, 2, 3]),
          (False, (7, 6, 5, 4), [0.3, 0.1, 0.2, 0.4, 0.05], [1, 2, 3, 4, 2]), (False, (300,), [0.7], [1]),
          (True, (40, 36), [0.3, 0.2], [1, 2]), (True, (12, 10, 8), [0.2, 0.3], [3, 3]), (True, (300,), [0.7], [1]),
          (True, (9, 8, 7), [0.4], [2])]


@pytest.mark.parametrize("it", [0, 4])
@pytest.mark.parametrize("case", PARITY, ids=["pd-2d", "pd-3d", "pd-4d-5terms", "pd-1d", "pd2-2d", "pd2-repeated", "pd2-1d", "pd2-1term"])
def test_host_forward_equals_oracle(port, prox, case, it):
    pd2, shp, ws, ds = case
    V = np.asfortranarray(np.random.default_rng(14).normal(size=shp))
    want, info = (port.pd2_tv if pd2 else port.pd_tv)(V, list(ws), ds, maxit=it)
    K = int(info[0])
    assert K >= 1
    got, passes = P.forward(prox, V.ravel(order="F"), shp, ws, ds, K, pd2)
    assert len(passes) == P.n_passes(pd2, len(ws), K)
    assert np.abs(got - want.ravel(order="F")).max() <= 1e-12 * np.abs(want).max(), (shp, it, K)


# (pd2, shape, ws, ds): 1D / 2D / 3D, 1 / 2 / 3 / 5 terms, a repeated axis, a zero penalty
CASES = [(False, (9,), [0.3], [1]),
         (False, (5, 6), [0.25, 0.35], [1, 2]),
         (False, (5, 6), [0.3, 0.0], [1, 2]),
         (False, (4, 3, 5), [0.2, 0.3, 0.15], [1, 2, 3]),
         (False, (3, 4, 3), [0.04, 0.02, 0.06, 0.03, 0.05], [1, 2, 3, 1, 2]),
         (True, (5, 6), [0.25, 0.35], [1, 2]),
         (True, (5, 6), [0.0, 0.3], [1, 2]),
         (True, (4, 3, 5), [0.2, 0.3], [3, 1])]
CASE_IDS = ["pd-1d", "pd-2d", "pd-2d-zero", "pd-3d", "pd-3d-5terms", "pd2-2d", "pd2-2d-zero", "pd2-3d"]
ONE_TERM_PD2 = [(True, (9,), [0.3], [1]), (True, (4, 3, 5), [0.2], [2])]


def fd_check(prox, case, K, seed):
    """Every element of y and every penalty (right derivative at a zero penalty) against the restatement."""
    pd2, ns, ws, ds = case
    y = volume(ns, seed).ravel(order="F")
    G = np.random.default_rng(5).normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, K, pd2)
    gY, glam = P.backward(passes, G, ns, ws, ds, K, pd2)
    f0 = objective(prox, y, ns, ws, ds, G, K, pd2)
    fd = np.empty_like(y)
    for e in range(y.size):
        def step(h):
            yh = y.copy(); yh[e] += h
            return objective(prox, yh, ns, ws, ds, G, K, pd2) - f0
        fd[e] = kink_free(step)
    check_close(fd, gY)
    fw = []
    for i in range(len(ws)):
        def step(h):
            if ws[i] == 0.0 and h < 0:
                return None
            wh = list(ws); wh[i] += h
            return objective(prox, y, ns, wh, ds, G, K, pd2) - f0
        fw.append(kink_free(step))
    check_close(fw, glam if pd2 else len(ws) * glam)      # PD_TV's ws_i is scaled to npen ws_i: its gradient is npen glam_i


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("K", [1, 2, 5, 35])
def test_elementwise(prox, case, K):
    fd_check(prox, case, K, 11 + K)


@pytest.mark.parametrize("case", ONE_TERM_PD2, ids=["1d", "3d"])
def test_elementwise_pd2_one_term(prox, case):
    """PD2_TV with one term runs exactly one iteration (one pass), whatever K is."""
    fd_check(prox, case, 1, 3)


@pytest.mark.parametrize("pd2", [False, True], ids=["pd", "pd2"])
@pytest.mark.parametrize("K", [2, 5, 35])
def test_directional(prox, pd2, K):
    """12 x 10 x 8: random directions in y, and the penalties one at a time (PD_TV with 3 terms, PD2_TV with 2)."""
    ns = (12, 10, 8)
    ws, ds = ([0.2, 0.3], [1, 3]) if pd2 else ([0.2, 0.3, 0.25], [1, 2, 3])
    y = volume(ns, 3 + K).ravel(order="F")
    rng = np.random.default_rng(17)
    G = rng.normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, K, pd2)
    gY, glam = P.backward(passes, G, ns, ws, ds, K, pd2)
    f0 = objective(prox, y, ns, ws, ds, G, K, pd2)
    for _ in range(2):
        V = rng.normal(size=y.size)
        check_close([kink_free(lambda e: objective(prox, y + e * V, ns, ws, ds, G, K, pd2) - f0)], [np.sum(gY * V)])
    fw = []
    for i in range(len(ws)):
        def step(e):
            wh = list(ws); wh[i] += e
            return objective(prox, y, ns, wh, ds, G, K, pd2) - f0
        fw.append(kink_free(step))
    check_close(fw, glam if pd2 else len(ws) * glam)


def test_zero_penalties():
    """Every penalty 0: every pass is the identity.  PD_TV after one iteration is the mean of the copies, and gY the same sum of G / kk;
    PD2_TV returns y, and gY = G."""
    y = volume((6, 5), 1).ravel(order="F")
    G = np.random.default_rng(2).normal(size=y.size)
    ident = lambda a, *_: a.copy()                                 # noqa: E731
    out, passes = P.forward(ident, y, (6, 5), [0.0] * 3, [1, 2, 1], 1, False)
    assert len(passes) == 3 and np.array_equal(out, ((0 + y / 3.0) + y / 3.0) + y / 3.0)
    gY, glam = P.backward(passes, G, (6, 5), [0.0] * 3, [1, 2, 1], 1, False)
    assert np.array_equal(gY, ((0 + (G / 3.0 - 0)) + (G / 3.0 - 0)) + (G / 3.0 - 0))
    out, passes = P.forward(ident, y, (6, 5), [0.0, 0.0], [1, 2], 4, True)
    assert len(passes) == 8 and np.array_equal(out, y)
    gY, _ = P.backward(passes, G, (6, 5), [0.0, 0.0], [1, 2], 4, True)
    assert np.allclose(gY, G, rtol=0, atol=1e-14)


@pytest.mark.parametrize("case", CASES + ONE_TERM_PD2 + [(False, (7, 1, 6), [0.3, 0.2, 0.4], [1, 2, 3])],
                         ids=CASE_IDS + ["pd2-1term-1d", "pd2-1term-3d", "pd-len1-axis"])
@pytest.mark.parametrize("K", [2, 35])
def test_tape_driven_restatement_equals_pass_driven(prox, case, K):
    pd2, ns, ws, ds = case
    y = np.round(volume(ns, 9) * 4) / 4                     # ties in the input
    y = y.ravel(order="F")
    G = np.random.default_rng(2).normal(size=y.size)
    _, passes = P.forward(prox, y, ns, ws, ds, K, pd2)
    tapes = P.pass_tapes(passes, ns, ws, ds, pd2)
    for dt in (np.float64, np.float32):
        Gt, pt = G.astype(dt), [X.astype(dt) for X in passes]
        want = P.backward(pt, Gt, ns, ws, ds, K, pd2)
        got = P.backward_from_tapes(P.pass_tapes(pt, ns, ws, ds, pd2) if dt == np.float32 else tapes, Gt, ns, ds, K, pd2)
        assert got[0].dtype == dt and np.array_equal(got[0], want[0])
        assert np.array_equal(got[1], want[1])


def test_tape_bytes_in_64_bits():
    """The tape sizes of the N-D solvers are computed in 64-bit arithmetic (a host function: no device needed).  A pass count past
    2^32 gives the exact size, and a size past 2^64 gives 0, which the record calls refuse."""
    import ctypes as C
    import proxtv_b200
    lib = proxtv_b200.load()
    sb2 = lambda n: 2 * (((n + 31) // 32 * 4 + 255) // 256 * 256)          # noqa: E731
    ns = np.array([20, 16, 12], dtype=np.int32)
    p = C.c_void_p(ns.ctypes.data)
    huge = 1431655766                                              # 3 huge = 2^32 + 2
    assert lib.proxtv_PD_TV_tape_bytes(p, 3, 3, huge) == 256 + 3 * huge * sb2(3840)
    assert lib.proxtv_PD2_TV_tape_bytes(p, 3, 2, huge) == 256 + 2 * huge * sb2(3840)
    assert lib.proxtv_PD2_TV_tape_bytes(p, 3, 1, huge) == 256 + sb2(3840)
    assert lib.proxtv_PDR_TV_tape_bytes(p, 3, 3, huge) == 256 + 3 * (huge - 1) * sb2(3840)
    big = np.array([1 << 15] * 3, dtype=np.int32)                  # 2^45 elements: 2^31 iterations x 64 terms of them pass 2^64 bytes
    pb = C.c_void_p(big.ctypes.data)
    top = 2 ** 31 - 1
    assert lib.proxtv_PD_TV_tape_bytes(pb, 3, 64, top) == 0
    assert lib.proxtv_PD2_TV_tape_bytes(pb, 3, 2, top) == 0
    assert lib.proxtv_PDR_TV_tape_bytes(pb, 3, 64, top) == 0
