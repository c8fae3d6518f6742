"""The backward pass of the weighted DR2L1W_TV on the host (DESIGN.md section 12), shared by test_drw_vjp_cpu.py and test_gpu_drw_vjp.py:

* ``forward`` -- DR2L1W_TV in float64 in the association of solver.cu: drw_device, every prox pass the oracle's weighted taut string
  (``Port.tv1_weighted``, bit-identical to the device's weighted kernels), recording all 2K + 2 pass outputs;
* ``backward`` -- the unrolled vector-Jacobian product of include/proxtv_b200.h (proxtv_DR2L1W_TV_vjp_dev_*) restated in numpy: per
  pass vjp_emu.restate under that pass's segmentation and weights, the combines in the storage type with the kernels' association,
  the start value term as a float64 sum, and each edge weight's gradient summed in float64 over the passes in backward order;
* ``backward_from_tapes`` -- the same restatement driven by decoded (F, U) segmentation tapes instead of pass outputs, so that float32
  and device tapes can be checked without a host float32 forward;
* ``pass_tapes`` / ``device_pass_tapes`` -- the (F, U) tapes of the host passes / of a device tape buffer.
Images are (M, N) arrays in natural layout: W1 (M-1, N) weights the edges along columns (w_col), W2 (M, N-1) along rows (w_row).
Pass p = 2k is the column pass of iteration k, p = 2k + 1 its row pass, k = K the final pair."""
import numpy as np

import dr2_vjp_emu as D
import vjp_emu

MAX_ITERS = 35


def _cols(port, A, W1):
    M, N = A.shape
    if M == 1:
        return A.copy()
    return np.stack([port.tv1_weighted(A[:, j], W1[:, j]) for j in range(N)], axis=1)


def _rows(port, A, W2):
    M, N = A.shape
    if N == 1:
        return A.copy()
    return np.stack([port.tv1_weighted(A[i], W2[i]) for i in range(M)], axis=0)


def forward(port, Y, W1, W2, maxit=0):
    """DR2L1W_TV of Y (M, N) float64; returns (out, passes) with passes the 2K + 2 pass outputs in execution order.  The start value
    is the float64 sum, doubled, divided by M N."""
    Y = np.asarray(Y, dtype=np.float64)
    M, N = Y.shape
    K = MAX_ITERS if maxit <= 0 else maxit
    t = np.full(Y.shape, (2.0 * Y.sum()) / float(M * N))
    passes = []
    for k in range(K + 1):
        final = k == K
        x1 = _cols(port, t, W1)
        passes.append(x1)
        d = t - x1
        s = d if final else 2.0 * d - t
        u = Y - s
        x2 = _rows(port, u, W2)
        passes.append(x2)
        tw = (u - x2) - Y
        if final:
            return -s - tw, passes
        t = 0.5 * (t + (-2.0 * tw - s))


def _run(S, G, K, shape1, shape2):
    """The recurrence of proxtv_b200/csrc/dr2_vjp.cu: drw_vjp_device; S(p, gin) -> (gx, gw) of pass p for the upstream gradient gin."""
    T = G.dtype.type
    M, N = G.shape
    acc1, acc2 = np.zeros(shape1), np.zeros(shape2)
    a, gw = S(2 * K + 1, G); acc2 = acc2 + gw.astype(np.float64)
    sc, gw = S(2 * K, a); acc1 = acc1 + gw.astype(np.float64)
    gY = a.copy()
    g = sc - a
    for k in range(K - 1, -1, -1):
        a, gw = S(2 * k + 1, g); acc2 = acc2 + gw.astype(np.float64)
        gY = gY + a
        h = g - T(2) * a
        sc, gw = S(2 * k, h); acc1 = acc1 + -1.0 * gw.astype(np.float64)
        g = (a + h) - sc
    gY = (gY.astype(np.float64) + (2.0 * g.astype(np.float64).sum()) / float(M * N)).astype(T)
    return gY, acc1.astype(T), acc2.astype(T)


def _S_cols(X, G, W1):
    gx, gw = vjp_emu.restate(np.ascontiguousarray(X.T), np.ascontiguousarray(G.T), 0.0, W=np.ascontiguousarray(W1.T))
    return np.ascontiguousarray(gx.T), np.ascontiguousarray(gw.T)


def _S_rows(X, G, W2):
    return vjp_emu.restate(np.ascontiguousarray(X), np.ascontiguousarray(G), 0.0, W=np.ascontiguousarray(W2))


def backward(passes, G, W1, W2, maxit=0):
    """(gY, gW1, gW2) in G's dtype for the upstream gradient G (M, N) of forward()'s output."""
    K = MAX_ITERS if maxit <= 0 else maxit
    T = G.dtype
    W1, W2 = np.asarray(W1, dtype=T), np.asarray(W2, dtype=T)

    def S(p, gin):
        X = passes[p].astype(T)
        return _S_cols(X, gin, W1) if p % 2 == 0 else _S_rows(X, gin, W2)
    return _run(S, G, K, W1.shape, W2.shape)


# ---------------------------------------------------------------------------------------------------------------- tapes
def _geom(M, N, col):
    """(nf, len, inc) of a pass over a column-major M x N image."""
    return (N, M, 1) if col else (M, N, M)


def pass_tapes(passes, W1, W2):
    """(F, U) of every host pass over the column-major image (the device's storage order)."""
    out = []
    for p, X in enumerate(passes):
        M, N = X.shape
        col = p % 2 == 0
        W = np.ascontiguousarray(W1.T) if col else np.asarray(W2)
        out.append(D.tape_bits(X.ravel(order="F"), *_geom(M, N, col), 0.0, W))
    return out


def device_pass_tapes(raw, M, N, maxit=0):
    """The 2K + 2 (F, U) pairs of a device tape buffer (uint8 numpy array, 256-byte header first)."""
    K = MAX_ITERS if maxit <= 0 else maxit
    nw = D.tape_words(M * N)
    words = np.asarray(raw)[256:256 + (2 * K + 2) * 2 * nw * 4].view(np.uint32).reshape(2 * K + 2, 2, nw)
    return [(words[p, 0], words[p, 1]) for p in range(2 * K + 2)]


def _bits(words, n):
    return ((words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(bool).ravel()[:n]


def _surrogate(F, U, M, N, col, T):
    """Fibers (nf, len) and weights (nf, len-1) that have the segmentation the tape (F, U) encodes: an integer staircase going up,
    down or level per edge (exact in any float type), weight 0 on the (1, 1) "equal with zero weight" edges, 1 elsewhere."""
    nf, ln, inc = _geom(M, N, col)
    idx = vjp_emu.flat_index(nf, ln, inc)[:, :-1]
    f, u = _bits(F, M * N)[idx], _bits(U, M * N)[idx]
    step = np.where(f, 0.0, np.where(u, 1.0, -1.0))
    Y = np.concatenate([np.zeros((nf, 1)), np.cumsum(step, axis=1)], axis=1).astype(T)
    W = np.where(f & u, 0.0, 1.0).astype(T)
    return Y, W


def backward_from_tapes(tapes, G, maxit=0):
    """backward() driven by the 2K + 2 (F, U) tapes (pass_tapes / device_pass_tapes) instead of the pass outputs."""
    K = MAX_ITERS if maxit <= 0 else maxit
    T = G.dtype.type
    M, N = G.shape

    def S(p, gin):
        col = p % 2 == 0
        Ys, Ws = _surrogate(tapes[p][0], tapes[p][1], M, N, col, T)
        if col:
            gx, gw = vjp_emu.restate(Ys, np.ascontiguousarray(gin.T), 0.0, W=Ws)
            return np.ascontiguousarray(gx.T), np.ascontiguousarray(gw.T)
        return vjp_emu.restate(Ys, np.ascontiguousarray(gin), 0.0, W=Ws)
    return _run(S, G, K, (M - 1, N), (M, N - 1))
