"""CPU tests of per-item penalties for the batched PD_TV / PD2_TV (DESIGN.md section 16.1), no GPU needed.

* A host restatement of the per-item solve: pd_vjp_emu's forward / backward driven per item with that item's own ws row and its own
  K_b.  Its backward -- gY of every item and the (B, npen) gradient of the per-item penalties -- matches central finite differences
  at fixed K_b on a batch whose items stop at different K, with an item whose penalties are all zero and one with a zero term.
* tvgen_batched's shape rules for a 2-D ws raise AssertionError before any device is needed; a 1-D ws keeps its meaning when B == npen.
* The per-item entry points and the per-fiber test entry points are in the header and the ctypes table (tests/test_abi.py compares
  the two); without a device they refuse and leave their outputs untouched.
"""
import ctypes as C

import numpy as np
import pytest

import pd_vjp_emu as P
import proxtv_b200
from test_drw_vjp_cpu import kink_free
from test_pd_batched_cpu import item_K, mixed_batch, prox  # noqa: F401  (prox: the module fixture)
from test_pdr_vjp_cpu import check_close


def items_forward(prox, Y, ns, W, ds, maxit, pd2):
    """(out (B, n), K): item b solved alone with its row W[b] and its own stop rule."""
    K = [item_K(prox, Y[b], ns, list(W[b]), ds, maxit, pd2) for b in range(Y.shape[0])]
    out = np.stack([P.forward(prox, Y[b], ns, list(W[b]), ds, K[b], pd2)[0] for b in range(Y.shape[0])])
    return out, K


def items_backward(prox, Y, G, ns, W, ds, K, pd2):
    """(gY (B, n), glam (B, npen) of each item's penalties as given)."""
    gY, glam = np.empty_like(G), np.zeros(W.shape)
    for b in range(Y.shape[0]):
        passes = P.forward(prox, Y[b], ns, list(W[b]), ds, K[b], pd2)[1]
        g, gl = P.backward(passes, G[b], ns, list(W[b]), ds, K[b], pd2)
        gY[b], glam[b] = g, gl * (1.0 if pd2 else W.shape[1])
    return gY, glam


@pytest.mark.parametrize("case", [(False, (5, 4), [[0.25, 0.1, 0.3], [0.0, 0.0, 0.0], [0.05, 0.4, 0.0]], [1, 2, 1]),
                                  (True, (5, 4), [[0.2, 0.3], [0.0, 0.0], [0.35, 0.0]], [1, 2])], ids=["pd", "pd2"])
def test_per_item_restatement_agrees_with_differences(prox, case):
    pd2, ns, W, ds = case
    W = np.array(W)
    Y = mixed_batch(ns)
    out, K = items_forward(prox, Y, ns, W, ds, 4, pd2)
    assert len(set(K)) >= 2, K                                     # the items stop at different K
    G = np.random.default_rng(8).normal(size=Y.shape)
    gY, glam = items_backward(prox, Y, G, ns, W, ds, K, pd2)

    def obj(Yh, Wh):
        return sum(float(np.sum(P.forward(prox, Yh[b], ns, list(Wh[b]), ds, K[b], pd2)[0] * G[b])) for b in range(Y.shape[0]))
    f0 = obj(Y, W)
    fd = np.empty_like(Y)
    for b in range(Y.shape[0]):
        for e in range(Y.shape[1]):
            def step(h):
                Yh = Y.copy(); Yh[b, e] += h
                return obj(Yh, W) - f0
            fd[b, e] = kink_free(step)
    check_close(fd, gY)
    fw = np.empty(W.shape)
    for b in range(W.shape[0]):
        for i in range(W.shape[1]):
            def step(h):
                if W[b, i] == 0.0 and h < 0:
                    return None
                Wh = W.copy(); Wh[b, i] += h
                return obj(Y, Wh) - f0
            fw[b, i] = kink_free(step)
    check_close(fw, glam)
    # an item's row only moves that item's gradient: the shared-ws gradient is the sum of the rows
    check_close(fw.sum(axis=0), glam.sum(axis=0))


def test_python_shape_rules_before_the_device(monkeypatch):
    def no_library(*a, **k):
        raise RuntimeError("the library was called")
    monkeypatch.setattr(proxtv_b200, "_host_call", no_library)
    x = np.zeros((3, 4, 4))
    bad = [np.full((2, 2), 0.1), np.full((3, 3), 0.1), np.full((3, 1), 0.1), np.full((4, 2), 0.1)]
    for w in bad + [w.tolist() for w in bad]:
        with pytest.raises(AssertionError):
            proxtv_b200.tvgen_batched(x, w, [1, 2], [1, 1])
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(np.zeros(4), np.full((4, 1), 0.1), [1], [1])     # items need x.ndim >= 2
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(x, np.full((3, 2), 0.1), [1, 2], [1, 1], max_iters=-1)
    with pytest.raises(NotImplementedError):
        proxtv_b200.tvgen_batched(x, np.full((3, 2), 0.1), [1, 2], [1, 2])
    # a (B, npen) ws that passes the checks reaches the per-item host entry; a 1-D ws of length B == npen stays shared
    seen = []
    monkeypatch.setattr(proxtv_b200, "_host_call", lambda name, *a, **k: seen.append((name, np.array(a[2]))))
    proxtv_b200.tvgen_batched(np.zeros((2, 4, 4)), [[0.1, 0.2], [0.3, 0.4]], [1, 2], [1, 1])
    proxtv_b200.tvgen_batched(np.zeros((2, 4, 4)), [0.1, 0.2], [1, 2], [1, 1])
    assert seen[0][0] == "PD2_TV_batched_items" and np.array_equal(seen[0][1], [0.1, 0.2, 0.3, 0.4])
    assert seen[1][0] == "PD2_TV_batched" and np.array_equal(seen[1][1], [0.1, 0.2])


def test_torch_shape_rules_before_the_device():
    torch = pytest.importorskip("torch")
    from proxtv_b200 import _nd_torch
    x = torch.zeros((3, 4, 4), dtype=torch.float64)          # CPU tensor: the device check would come later, the shapes fail first
    with pytest.raises(AssertionError):
        _nd_torch("PD2_TV", proxtv_b200.tvgen_batched, x, [0.1] * 6, torch.zeros(2, 3), [1, 2], 0, batched=True, items=True)
    with pytest.raises(AssertionError):
        _nd_torch("PD2_TV", proxtv_b200.tvgen_batched, x, [0.1] * 4, None, [1, 2], 0, batched=True, items=True)
    with pytest.raises(AssertionError):
        proxtv_b200.tvgen_batched(x, torch.zeros(2, 2), [1, 2], [1, 1])


@pytest.mark.skipif(proxtv_b200.load().proxtv_device_count() != 0, reason="a CUDA device is present")
def test_items_entry_points_fail_loudly_without_device():
    lib = proxtv_b200.load()
    x = np.random.default_rng(0).normal(size=(3, 6, 5))
    y = np.ascontiguousarray(x); out = np.full_like(y, -7.0); info = np.zeros(9)
    ns = np.array([5, 6], dtype=np.int32); lam = np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6]); dims = np.array([1.0, 2.0])
    a = lambda v: C.c_void_p(v.ctypes.data)                                # noqa: E731
    for f in (lib.proxtv_PD2_TV_batched_items_f64, lib.proxtv_PD_TV_batched_items_f64):
        info[:] = 0
        assert f(a(y), a(lam), a(dims), a(out), a(info), a(ns), 2, 2, 3, 0) == 0
        assert np.all(out == -7.0) and np.all(info[2::3] == 3) and np.all(info[0::3] == 0)
        assert np.array_equal(lam, [0.1, 0.2, 0.3, 0.4, 0.5, 0.6])
    # the per-fiber prox refuses its groups before it looks for a device
    tab = np.array([0.1, 0.2])
    for fpi in (0, 4):
        assert lib.proxtv_prox_fibers_lamf_dev_f64(a(y), a(out), 6, 5, 1, a(tab), fpi, None) == 0
        assert b"penalty groups" in lib.proxtv_last_error()
    assert lib.proxtv_prox_fibers_lamf_dev_f64(a(y), a(out), 6, 5, 1, None, 3, None) == 0
    assert b"NULL" in lib.proxtv_last_error()
