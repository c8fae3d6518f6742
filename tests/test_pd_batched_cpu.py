"""CPU tests of the batched PD_TV / PD2_TV (DESIGN.md section 16), no GPU needed.

* A host restatement of the batched solve: the slot rule (at iteration j the items {b : K_b > j} in increasing b), each item's K_b
  from its own stop rule, and pd_vjp_emu's forward / backward driven per item with K_b, unmodified.  It agrees with a loop over the
  items, and its backward -- gY of every item and the gradient of the shared penalties, the per-item sums -- matches finite differences
  at fixed K_b on a small mixed batch whose items stop at different K, with one zero penalty term.
* The batched tape sizes: the capacity formula, in 64-bit arithmetic, 0 on overflow or invalid arguments.
* tvgen_batched's assertions and NotImplementedError for p != 1 come before any device is needed; without a device the calls raise
  ProxTVError and the raw C ABI leaves its outputs untouched with RC_ERROR.
"""
import ctypes as C

import numpy as np
import pytest

import pd_vjp_emu as P
import proxtv_b200
from pdr_vjp_emu import exact_prox
from test_drw_vjp_cpu import kink_free
from test_pdr_vjp_cpu import check_close, volume

STOP_PD = 1e-6


@pytest.fixture(scope="module")
def prox(port):
    return exact_prox(port)


def slots(K, j):
    """The slot rule: the items running at iteration j, in slot order."""
    return [b for b in range(len(K)) if K[b] > j]


def item_K(prox, y, ns, ws, ds, maxit, pd2):
    """An item's own K: the first iteration count whose stop value mean|x_K - x_{K-1}| is <= 1e-6, or the cap."""
    cap = 1 if pd2 and len(ws) == 1 else maxit
    prev = y.copy() if pd2 else np.zeros_like(y)                    # PD2_TV starts from x = y, PD_TV from x = 0
    for K in range(1, cap + 1):
        x = P.forward(prox, y, ns, ws, ds, K, pd2)[0]
        if np.mean(np.abs(x - prev)) <= STOP_PD:
            return K
        prev = x
    return cap


def batched_forward(prox, Y, ns, ws, ds, maxit, pd2):
    """(out (B, n), K) of the batched solve: the running items of every iteration by the slot rule, each item's x leaving at its K."""
    B = Y.shape[0]
    K = [item_K(prox, Y[b], ns, ws, ds, maxit, pd2) for b in range(B)]
    out = np.full_like(Y, np.nan)
    for j in range(max(K)):
        for b in slots(K, j):
            if K[b] == j + 1:                                       # stops after this iteration
                out[b] = P.forward(prox, Y[b], ns, ws, ds, K[b], pd2)[0]
    return out, K


def batched_backward(prox, Y, G, ns, ws, ds, K, pd2):
    """(gY (B, n), glam (B, npen) of the penalties as given): items join the backward at j = K_b - 1, from the largest K down."""
    B = Y.shape[0]
    gY, glam = np.full_like(G, np.nan), np.zeros((B, len(ws)))
    joined = []
    for j in range(max(K) - 1, -1, -1):
        for b in slots(K, j):
            if b in joined:
                continue
            joined.append(b)
            passes = P.forward(prox, Y[b], ns, ws, ds, K[b], pd2)[1]
            g, gl = P.backward(passes, G[b], ns, ws, ds, K[b], pd2)
            gY[b], glam[b] = g, gl * (1.0 if pd2 else len(ws))
    assert sorted(joined) == list(range(B))
    return gY, glam


def mixed_batch(ns):
    n = int(np.prod(ns))
    return np.stack([volume(ns, 3).ravel(order="F"), np.full(n, 0.4), volume(ns, 4).ravel(order="F")])


def test_slot_rule():
    K = [3, 1, 5, 3, 2]
    assert slots(K, 0) == [0, 1, 2, 3, 4]
    assert slots(K, 1) == [0, 2, 3, 4]
    assert slots(K, 2) == [0, 2, 3]
    assert slots(K, 4) == [2]
    assert slots(K, 5) == []


@pytest.mark.parametrize("case", [(False, (5, 4), [0.25, 0.0, 0.3], [1, 2, 1]), (True, (5, 4), [0.0, 0.3], [1, 2])],
                         ids=["pd", "pd2"])
def test_restatement_agrees_with_loop_and_differences(prox, case):
    pd2, ns, ws, ds = case
    Y = mixed_batch(ns)
    maxit = 4
    out, K = batched_forward(prox, Y, ns, ws, ds, maxit, pd2)
    assert len(set(K)) >= 2, K                                     # the items stop at different K
    for b in range(Y.shape[0]):
        assert np.array_equal(out[b], P.forward(prox, Y[b], ns, ws, ds, K[b], pd2)[0])
    G = np.random.default_rng(6).normal(size=Y.shape)
    gY, glam = batched_backward(prox, Y, G, ns, ws, ds, K, pd2)

    def obj(Yh, wh):
        return sum(float(np.sum(P.forward(prox, Yh[b], ns, wh, ds, K[b], pd2)[0] * G[b])) for b in range(Y.shape[0]))
    f0 = obj(Y, ws)
    fd = np.empty_like(Y)
    for b in range(Y.shape[0]):
        for e in range(Y.shape[1]):
            def step(h):
                Yh = Y.copy(); Yh[b, e] += h
                return obj(Yh, ws) - f0
            fd[b, e] = kink_free(step)
    check_close(fd, gY)
    fw = []
    for i in range(len(ws)):
        def step(h):
            if ws[i] == 0.0 and h < 0:
                return None
            wh = list(ws); wh[i] += h
            return obj(Y, wh) - f0
        fw.append(kink_free(step))
    check_close(fw, glam.sum(axis=0))


def test_batched_tape_bytes():
    lib = proxtv_b200.load()
    sb2 = lambda n: 2 * (((n + 31) // 32 * 4 + 255) // 256 * 256)          # noqa: E731
    head = lambda B: 256 + (4 * B + 255) // 256 * 256                      # noqa: E731
    ns = np.array([20, 16, 12], dtype=np.int32)
    p = C.c_void_p(ns.ctypes.data)
    for B in (1, 7, 100):
        assert lib.proxtv_PD_TV_batched_tape_bytes(p, 3, 3, B, 0) == head(B) + 35 * 3 * sb2(3840 * B)
        assert lib.proxtv_PD2_TV_batched_tape_bytes(p, 3, 2, B, 10) == head(B) + 20 * sb2(3840 * B)
        assert lib.proxtv_PD2_TV_batched_tape_bytes(p, 3, 1, B, 10) == head(B) + sb2(3840 * B)
    huge = 1431655766                                              # 3 huge = 2^32 + 2 passes
    assert lib.proxtv_PD_TV_batched_tape_bytes(p, 3, 3, 2, huge) == head(2) + 3 * huge * sb2(7680)
    big = np.array([1 << 15] * 3, dtype=np.int32)
    pb = C.c_void_p(big.ctypes.data)
    assert lib.proxtv_PD_TV_batched_tape_bytes(pb, 3, 64, 4, 2 ** 31 - 1) == 0
    assert lib.proxtv_PD2_TV_batched_tape_bytes(pb, 3, 2, 2 ** 31 - 1, 2 ** 31 - 1) == 0
    assert lib.proxtv_PD_TV_batched_tape_bytes(p, 3, 3, 0, 5) == 0         # batch < 1
    assert lib.proxtv_PD2_TV_batched_tape_bytes(p, 3, 3, 2, 5) == 0        # PD2_TV takes 1 or 2 terms
    assert lib.proxtv_PD_TV_batched_tape_bytes(None, 3, 3, 2, 5) == 0


def test_python_surface_checks_before_the_device():
    x = np.zeros((2, 4, 4))
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(x, [0.1], [1, 2], [1])
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(x, [0.1, 0.1], [1, 2], [1])
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(x, [0.1], [1], [1], max_iters=-1)
    with pytest.raises(NotImplementedError):
        proxtv_b200.tvgen_batched(x, [0.1, 0.2], [1, 2], [1, 2])
    assert "tvgen_batched" in proxtv_b200.__all__


@pytest.mark.skipif(proxtv_b200.load().proxtv_device_count() != 0, reason="a CUDA device is present")
def test_fails_loudly_without_device():
    x = np.random.default_rng(0).normal(size=(3, 6, 5))
    with pytest.raises(proxtv_b200.ProxTVError):
        proxtv_b200.tvgen_batched(x, [0.1, 0.2, 0.1], [1, 2, 1], [1, 1, 1])
    lib = proxtv_b200.load()
    y = np.ascontiguousarray(x); out = np.full_like(y, -7.0); info = np.zeros(9)
    ns = np.array([5, 6], dtype=np.int32); lam = np.array([0.1, 0.2]); dims = np.array([1.0, 2.0])
    a = lambda v: C.c_void_p(v.ctypes.data)                                # noqa: E731
    for f in (lib.proxtv_PD2_TV_batched_f64, lib.proxtv_PD_TV_batched_f64):
        info[:] = 0
        assert f(a(y), a(lam), a(dims), a(out), a(info), a(ns), 2, 2, 3, 0) == 0
        assert np.all(out == -7.0) and np.all(info[2::3] == 3) and np.all(info[0::3] == 0)
        assert np.array_equal(lam, [0.1, 0.2])
