"""The backward pass of the N-D PDR_TV on the host (DESIGN.md section 13), shared by test_pdr_vjp_cpu.py and test_gpu_pdr_vjp.py:

* ``forward`` -- PDR_TV in the storage type in the association of solver.cu (pdr_device, k_pdr_combine), every prox pass a chosen 1D
  solver over the fibers of one axis: ``exact_prox(port)`` (the oracle's linearized taut string per fiber, bit-identical to the device's
  sequential and chunked kernels in float64) or ``slope_prox(emu)`` (lane_emu.slope_fibers, the lane engine's plain pass), recording the
  (K - 1) npen pass outputs that reach the result;
* ``backward`` -- the unrolled vector-Jacobian product of include/proxtv_b200.h (proxtv_PDR_TV_vjp_dev_*) restated in numpy: per pass
  vjp_emu.restate under that pass's segmentation, the combines in the storage type with the kernels' association, and the penalty
  gradients summed in float64 over the passes in backward order;
* ``backward_from_tapes`` -- the same restatement driven by decoded (F, U) segmentation tapes instead of pass outputs;
* ``pass_tapes`` / ``device_pass_tapes`` -- the (F, U) tapes of the host passes / of a device tape buffer.
Arrays are column-major (the solver's storage order): a flat array of n = prod(ns) elements, axis a (1-based) has the fibers
``geom(ns, a)``.  Pass p = j npen + i is term i's pass of iteration j."""
import numpy as np

import dr2_vjp_emu as D
import vjp_emu
from lane_emu import slope_fibers

MAX_ITERS = 35


def geom(ns, d):
    """(nf, len, inc) of the fibers along the 1-based axis d of a column-major array of dims ns (solver.cu: geom_of)."""
    a = int(d) - 1
    n = int(np.prod(ns, dtype=np.int64))
    ln = int(ns[a])
    return (n // ln if ln else 0), ln, int(np.prod(ns[:a], dtype=np.int64))


def exact_prox(port):
    def prox(a, nf, ln, inc, lam):
        if lam == 0 or ln <= 1 or nf == 0:
            return a.copy()
        F = vjp_emu.from_flat(a, nf, ln, inc)
        return vjp_emu.to_flat(np.stack([port.tv1_linearized(F[j], float(lam)) for j in range(nf)]).astype(a.dtype), inc)
    return prox


def slope_prox(emu):
    def prox(a, nf, ln, inc, lam):
        return slope_fibers(emu, a, nf, ln, inc, lam)
    return prox


def scaled(ws, T):
    """The penalties the passes use: lambdas[i] *= npen in float64 (as run_pd), rounded to the storage type."""
    k = len(ws)
    return [T(float(w) * k) for w in ws]


def forward(prox, y, ns, ws, ds, maxit=0):
    """PDR_TV of the flat column-major array y (dims ns) in y's dtype; returns (out, passes), out flat like y."""
    T = y.dtype.type
    k = len(ws)
    kk = T(k)
    K = MAX_ITERS if maxit <= 0 else maxit
    lam = scaled(ws, T)
    z = [y.copy() for _ in range(k)]
    passes = []
    for j in range(K):
        p = [prox(z[i], *geom(ns, ds[i]), lam[i]) for i in range(k)]
        if j < K - 1:
            passes.extend(p)
        q = np.zeros_like(y)
        x = np.zeros_like(y)
        for i in range(k):
            q = q + p[i] / kk
            x = x + z[i] / kk
        for i in range(k):
            z[i] = z[i] + ((T(2) * q - x) - p[i])
    return x, passes


def _run(S, G, k, K):
    """The recurrence of proxtv_b200/csrc/dr2_vjp.cu: pdr_vjp_device; S(p, i, h) -> (gx, gw) of pass p (term i) for the upstream h."""
    T = G.dtype.type
    kk = T(k)
    v = G / kk
    gz = [v.copy() for _ in range(k)]
    glam = np.zeros(k)
    for j in range(K - 2, -1, -1):
        s = gz[0]
        for i in range(1, k):
            s = s + gz[i]
        sk = s / kk
        for i in range(k):
            h = T(2) * sk - gz[i]
            sc, gw = S(j * k + i, i, h)
            glam[i] += gw.astype(np.float64).sum()
            gz[i] = (gz[i] - sk) + sc
    gY = gz[0]
    for i in range(1, k):
        gY = gY + gz[i]
    return gY, glam


def backward(passes, G, ns, ws, ds, maxit=0):
    """(gY flat like G, glam float64 (npen,): the gradients of the scaled penalties) for the upstream gradient G (flat, storage type)
    of forward()'s output."""
    K = MAX_ITERS if maxit <= 0 else maxit
    k = len(ws)
    lam = scaled(ws, G.dtype.type)

    def S(p, i, h):
        nf, ln, inc = geom(ns, ds[i])
        X = passes[p].astype(G.dtype)
        gx, gw = vjp_emu.restate(vjp_emu.from_flat(X, nf, ln, inc), vjp_emu.from_flat(h, nf, ln, inc), lam[i])
        return vjp_emu.to_flat(gx, inc), gw
    return _run(S, G, k, K)


# ---------------------------------------------------------------------------------------------------------------- tapes
def pass_tapes(passes, ns, ws, ds):
    """(F, U) of every host pass."""
    k = len(ws)
    lam = scaled(ws, np.float64)
    return [D.tape_bits(X, *geom(ns, ds[p % k]), lam[p % k]) for p, X in enumerate(passes)]


def device_pass_tapes(raw, n, npen, maxit=0):
    """The (K - 1) npen (F, U) pairs of a device tape buffer (uint8 numpy array, 256-byte header first) of n-element passes."""
    K = MAX_ITERS if maxit <= 0 else maxit
    P = (K - 1) * npen
    nw = D.tape_words(n)
    words = np.asarray(raw)[256:256 + P * 2 * nw * 4].view(np.uint32).reshape(P, 2, nw)
    return [(words[p, 0], words[p, 1]) for p in range(P)]


def _bits(words, n):
    return ((words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(bool).ravel()[:n]


def surrogate(F, U, nf, ln, inc, T):
    """Fibers (nf, len) and weights (nf, len-1) with the segmentation the tape (F, U) encodes: an integer staircase going up, down or
    level per edge (exact in any float type), weight 0 on the (1, 1) "equal with zero weight" edges, 1 elsewhere."""
    n = nf * ln
    idx = vjp_emu.flat_index(nf, ln, inc)[:, :-1]
    f, u = _bits(F, n)[idx], _bits(U, n)[idx]
    step = np.where(f, 0.0, np.where(u, 1.0, -1.0))
    Y = np.concatenate([np.zeros((nf, 1)), np.cumsum(step, axis=1)], axis=1).astype(T)
    W = np.where(f & u, 0.0, 1.0).astype(T)
    return Y, W


def backward_from_tapes(tapes, G, ns, ds, maxit=0):
    """backward() driven by the (K - 1) npen (F, U) tapes (pass_tapes / device_pass_tapes) instead of the pass outputs."""
    K = MAX_ITERS if maxit <= 0 else maxit
    k = len(ds)
    T = G.dtype.type

    def S(p, i, h):
        nf, ln, inc = geom(ns, ds[i])
        Ys, Ws = surrogate(tapes[p][0], tapes[p][1], nf, ln, inc, T)
        gx, gw = vjp_emu.restate(Ys, vjp_emu.from_flat(h, nf, ln, inc), 0.0, W=Ws)
        return vjp_emu.to_flat(gx, inc), gw
    return _run(S, G, k, K)
